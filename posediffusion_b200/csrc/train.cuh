// Training kernels of the denoiser (csrc/api_train.cu): p_losses forward with saved activations, and its backward.
// Projections run on the tensor-core linear layer (tc_linear.cuh); everything here is fp32 element-wise, LayerNorm,
// attention and reduction code that only the denoiser uses: dropout, the schedule, the time MLP, the feed row, attention, the
// tail and the _first / time-MLP gradients.  What the backbone's training path needs too (LayerNorm, transposes, column sums,
// the linear-layer backward) is in csrc/train_common.cuh, with the rules that make gradients bit-identical from run to run.
#pragma once
#include <cstdint>

#include "posediff_b200.h"
#include "train_common.cuh"

namespace pdb {

constexpr int kTrainMaxFrames = 64;  // attention backward keeps Q, K, V, dO and two N x N tiles of one (sequence, head) in smem
constexpr int kFeedPad = 704;        // 702 feed columns (harmonic | t-embedding | z | pivot) zero-padded to a multiple of 64

// ---- dropout: Philox4x32-10 keyed by the 64-bit seed, counter = (element >> 2, element >> 34, layer << 8 | site, 0) ------------
// The same function builds the masks in the forward kernels, the backward kernels (masks are recomputed, never stored) and
// pdb_dropout_mask_host.  Element e is kept when word e & 3 of its block is >= threshold = floor(p * 2^32).
struct Philox4 {
  uint32_t v[4];
};
__host__ __device__ inline Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  Philox4 out = {{c0, c1, c2, c3}};
  return out;
}
__host__ __device__ inline uint32_t dropout_threshold(float p) {
  const double t = (double)p * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}
__host__ __device__ inline bool dropout_keep(uint64_t seed, int layer, int site, uint64_t e, uint32_t threshold) {
  if (threshold == 0) return true;
  const Philox4 r = philox4x32_10((uint32_t)(e >> 2), (uint32_t)(e >> 34), ((uint32_t)layer << 8) | (uint32_t)site, 0u,
                                  (uint32_t)seed, (uint32_t)(seed >> 32));
  return r.v[e & 3] >= threshold;
}
enum DropSite { kSiteAttn = 0, kSiteOut = 1, kSiteRelu = 2, kSiteFF2 = 3 };

struct DropCfg {
  uint64_t seed;
  uint32_t threshold;
  float scale;  // 1 / (1 - p)
};

// DDPM coefficients of the released schedule, float32 as GaussianDiffusion's buffers hold them:
// {sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod, sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod}
struct TrainSched {
  float c[PDB_NUM_TIMESTEPS][4];
};

}  // namespace pdb

namespace {
using namespace pdb;

// ---- forward -----------------------------------------------------------------------------------------------------------------
// time MLP per sequence: [cos(t f) | sin(t f)] -> Linear(256,128) -> SiLU -> Linear(128,128).  One block of 128 threads per sequence.
__global__ void train_time_mlp_kernel(const int* __restrict__ t, const float* __restrict__ w1, const float* __restrict__ b1,
                                      const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ u1,
                                      float* __restrict__ temb) {
  __shared__ float tf[256], s1[128];
  const int b = blockIdx.x, j = threadIdx.x;
  const float freq = expf(-logf(10000.0f) * (float)j / 128.0f);
  const float arg = (float)t[b] * freq;
  tf[j] = cosf(arg);
  tf[128 + j] = sinf(arg);
  __syncthreads();
  float a = b1[j];
  for (int k = 0; k < 256; ++k) a = fmaf(w1[j * 256 + k], tf[k], a);
  u1[b * 128 + j] = a;
  s1[j] = a / (1.0f + expf(-a));
  __syncthreads();
  float o = b2[j];
  for (int k = 0; k < 128; ++k) o = fmaf(w2[j * 128 + k], s1[k], o);
  temb[b * 128 + j] = o;
}

// q_sample + feed row: x_t = sqrt(abar_t) x_start + sqrt(1 - abar_t) noise (products rounded separately, as torch evaluates them);
// feed = [sin(x_t 2^k) | cos(x_t 2^k) | x_t | t-embedding | z | pivot one-hot | 0 0].
// kFromX (Denoiser.forward): the row is built from the given x_start = x itself; noise and x_t are not read or written.
template <bool kFromX>
__global__ void train_feed_kernel(const __grid_constant__ TrainSched sc, const float* __restrict__ x_start, const float* __restrict__ noise,
                                  const int* __restrict__ t, const float* __restrict__ temb, const float* __restrict__ z, int frames,
                                  int S, float* __restrict__ x_t, float* __restrict__ feed) {
  const int s = blockIdx.x;
  if (s >= S) return;
  const int b = s / frames, n = s - b * frames, tb = t[b];
  __shared__ float xs[9];
  if (threadIdx.x < 9) {
    if (kFromX) {
      xs[threadIdx.x] = x_start[s * 9 + threadIdx.x];
    } else {
      const float v = __fadd_rn(__fmul_rn(sc.c[tb][0], x_start[s * 9 + threadIdx.x]), __fmul_rn(sc.c[tb][1], noise[s * 9 + threadIdx.x]));
      xs[threadIdx.x] = v;
      x_t[s * 9 + threadIdx.x] = v;
    }
  }
  __syncthreads();
  float* row = feed + (size_t)s * kFeedPad;
  for (int col = threadIdx.x; col < kFeedPad; col += blockDim.x) {
    float v;
    if (col < 180) {
      const int j = col < 90 ? col : col - 90;
      const float arg = xs[j / 10] * (float)(1 << (j % 10));
      v = col < 90 ? sinf(arg) : cosf(arg);
    } else if (col < 189) {
      v = xs[col - 180];
    } else if (col < 317) {
      v = temb[b * 128 + col - 189];
    } else if (col < 701) {
      v = z[(size_t)s * 384 + col - 317];
    } else if (col == 701) {
      v = n == 0 ? 1.f : 0.f;
    } else {
      v = 0.f;
    }
    row[col] = v;
  }
}

// out = (res ? res : 0) + a * keep * scale * (gate ? gate > 0 : 1) over an [S, cols] array; mask element = flat index
__global__ void train_dropout_kernel(const float* a, const float* res, const float* gate, float* out, long long n, DropCfg d, int layer,
                                     int site) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = dropout_keep(d.seed, layer, site, (uint64_t)i, d.threshold) ? a[i] * d.scale : 0.f;
  if (gate && !(gate[i] > 0.f)) v = 0.f;
  out[i] = res ? res[i] + v : v;
}

// Self-attention of one (sequence, head): softmax(q k^T / sqrt(128)) with the probabilities saved (before dropout), dropout on the
// probabilities, then P v.  Warp per query row, lane per key for the scores, lane per column for P v.
__global__ void __launch_bounds__(256) train_attn_fwd_kernel(const float* __restrict__ qkv, int frames, DropCfg d, int layer,
                                                             float* __restrict__ P, float* __restrict__ att) {
  extern __shared__ float sm[];
  constexpr int LD = 129;
  const int N = frames, bh = blockIdx.x, b = bh / 4, h = bh % 4;
  float* Ks = sm;
  float* Vs = Ks + N * LD;
  float* qrow = Vs + N * LD;  // [8][128]
  float* prow = qrow + 8 * 128;  // [8][64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < N * 128; i += blockDim.x) {
    const int j = i >> 7, c = i & 127;
    const float* r = qkv + (size_t)(b * N + j) * 1536 + h * 128 + c;
    Ks[j * LD + c] = r[512];
    Vs[j * LD + c] = r[1024];
  }
  __syncthreads();
  const float scale = 0.08838834764831845f;  // 1 / sqrt(128)
  for (int i = warp; i < N; i += 8) {
    const float* qr = qkv + (size_t)(b * N + i) * 1536 + h * 128;
    for (int c = lane; c < 128; c += 32) qrow[warp * 128 + c] = qr[c];
    __syncwarp();
    float sc[2], mx = -INFINITY;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int j = lane + 32 * m;
      float s = -INFINITY;
      if (j < N) {
        s = 0.f;
        for (int c = 0; c < 128; ++c) s = fmaf(qrow[warp * 128 + c], Ks[j * LD + c], s);
        s *= scale;
      }
      sc[m] = s;
      mx = fmaxf(mx, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      sc[m] = (lane + 32 * m < N) ? expf(sc[m] - mx) : 0.f;
      sum += sc[m];
    }
    const float inv = 1.0f / warp_sum(sum);
    const size_t prow_base = ((size_t)bh * N + i) * N;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int j = lane + 32 * m;
      if (j < N) {
        const float p = sc[m] * inv;
        P[prow_base + j] = p;
        prow[warp * 64 + j] = dropout_keep(d.seed, layer, kSiteAttn, prow_base + j, d.threshold) ? p * d.scale : 0.f;
      }
    }
    __syncwarp();
    for (int c = lane; c < 128; c += 32) {
      float o = 0.f;
      for (int j = 0; j < N; ++j) o = fmaf(prow[warp * 64 + j], Vs[j * LD + c], o);
      att[(size_t)(b * N + i) * 512 + h * 128 + c] = o;
    }
    __syncwarp();
  }
}

// tail: LayerNorm(128) -> ReLU -> Linear(128, 9) -> eps; x_0_pred and the element-wise loss (reduction "none").  Warp per token.
// kEps (Denoiser.forward): eps itself is written to `loss`; x_t, noise, diff and x0 are not touched.
template <bool kEps>
__global__ void train_tail_fwd_kernel(const __grid_constant__ TrainSched sc, const float* __restrict__ u, const float* __restrict__ g,
                                      const float* __restrict__ bta, const float* __restrict__ w3, const float* __restrict__ b3,
                                      const int* __restrict__ t, const float* __restrict__ x_t, const float* __restrict__ noise, int frames,
                                      int S, int l2, float* __restrict__ stats, float* __restrict__ r, float* __restrict__ diff,
                                      float* __restrict__ loss, float* __restrict__ x0) {
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (s >= S) return;
  float v[4], mean, rstd;
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = u[(size_t)s * 128 + lane + 32 * i];
  ln_row_stats(v, 1e-5f, mean, rstd);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    v[i] = fmaxf((v[i] - mean) * rstd * g[c] + bta[c], 0.f);
    r[(size_t)s * 128 + c] = v[i];
  }
  if (lane == 0) {
    stats[2 * s] = mean;
    stats[2 * s + 1] = rstd;
  }
  const int tb = t[s / frames];
  for (int o = 0; o < 9; ++o) {
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) a = fmaf(w3[o * 128 + lane + 32 * i], v[i], a);
    const float eps = warp_sum(a) + b3[o];
    if (kEps) {
      if (lane == 0) loss[s * 9 + o] = eps;
    } else if (lane == 0) {
      const int e = s * 9 + o;
      x0[e] = __fsub_rn(__fmul_rn(sc.c[tb][2], x_t[e]), __fmul_rn(sc.c[tb][3], eps));
      const float dd = eps - noise[e];
      diff[e] = dd;
      loss[e] = l2 ? dd * dd : fabsf(dd);
    }
  }
}

// ---- backward ----------------------------------------------------------------------------------------------------------------
// tail backward, one warp per token: deps = grad_loss * dloss/deps - sqrt_recipm1(t) * grad_x0 (stored [S,9] for the _last.3
// gradients); dr = deps W3; d(LN out) = dr * (r > 0).  kEps (Denoiser.forward's backward): deps = grad_loss = dL/deps.
template <bool kEps>
__global__ void train_tail_bwd_kernel(const __grid_constant__ TrainSched sc, const float* __restrict__ diff, const float* __restrict__ gl,
                                      const float* __restrict__ gx0, const int* __restrict__ t, int frames, int S, int l2,
                                      const float* __restrict__ w3, const float* __restrict__ r, float* __restrict__ deps,
                                      float* __restrict__ dau) {
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (s >= S) return;
  const float cx = sc.c[t[s / frames]][3];
  float de[9];
#pragma unroll
  for (int o = 0; o < 9; ++o) {
    const int e = s * 9 + o;
    if (kEps) {
      de[o] = gl[e];
      continue;
    }
    const float dd = diff[e];
    const float dl = l2 ? 2.0f * dd : (float)((dd > 0.f) - (dd < 0.f));
    float v = gl ? gl[e] * dl : 0.f;
    if (gx0) v -= cx * gx0[e];
    de[o] = v;
  }
  if (lane < 9) deps[s * 9 + lane] = de[lane];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    float a = 0.f;
#pragma unroll
    for (int o = 0; o < 9; ++o) a = fmaf(de[o], w3[o * 128 + c], a);
    dau[(size_t)s * 128 + c] = r[(size_t)s * 128 + c] > 0.f ? a : 0.f;
  }
}

// _last.3 weight gradient partials: partial[chunk][o * 128 + k] = sum over the chunk's tokens of deps[s][o] r[s][k]
__global__ void train_w3_partial_kernel(const float* __restrict__ deps, const float* __restrict__ r, int S, float* __restrict__ partial) {
  const int k = threadIdx.x, chunk = blockIdx.x;
  const int per = (S + kRedChunks - 1) / kRedChunks, s0 = chunk * per, s1 = min(S, s0 + per);
  float acc[9] = {};
  for (int s = s0; s < s1; ++s) {
    const float rv = r[(size_t)s * 128 + k];
#pragma unroll
    for (int o = 0; o < 9; ++o) acc[o] = fmaf(deps[s * 9 + o], rv, acc[o]);
  }
#pragma unroll
  for (int o = 0; o < 9; ++o) partial[(size_t)chunk * 1152 + o * 128 + k] = acc[o];
}

// attention backward of one (sequence, head); writes the q / k / v column blocks of dqkv [S, 1536]
__global__ void __launch_bounds__(256) train_attn_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ P,
                                                             const float* __restrict__ datt, int frames, DropCfg d, int layer,
                                                             float* __restrict__ dqkv) {
  extern __shared__ float sm[];
  constexpr int LD = 129;
  const int N = frames, bh = blockIdx.x, b = bh / 4, h = bh % 4;
  const int LDN = N + 1;
  float* Qs = sm;
  float* Ks = Qs + N * LD;
  float* Vs = Ks + N * LD;
  float* Gs = Vs + N * LD;     // dO
  float* dS = Gs + N * LD;     // [N][N+1]
  float* Pd = dS + N * LDN;    // [N][N+1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < N * 128; i += blockDim.x) {
    const int j = i >> 7, c = i & 127;
    const float* r = qkv + (size_t)(b * N + j) * 1536 + h * 128 + c;
    Qs[j * LD + c] = r[0];
    Ks[j * LD + c] = r[512];
    Vs[j * LD + c] = r[1024];
    Gs[j * LD + c] = datt[(size_t)(b * N + j) * 512 + h * 128 + c];
  }
  __syncthreads();
  const float scale = 0.08838834764831845f;
  for (int i = warp; i < N; i += 8) {
    const size_t prow_base = ((size_t)bh * N + i) * N;
    float p[2], dp[2], dot = 0.f;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int j = lane + 32 * m;
      p[m] = dp[m] = 0.f;
      if (j < N) {
        float a = 0.f;
        for (int c = 0; c < 128; ++c) a = fmaf(Gs[i * LD + c], Vs[j * LD + c], a);
        const bool keep = dropout_keep(d.seed, layer, kSiteAttn, prow_base + j, d.threshold);
        p[m] = P[prow_base + j];
        dp[m] = keep ? a * d.scale : 0.f;
        Pd[i * LDN + j] = keep ? p[m] * d.scale : 0.f;
        dot = fmaf(p[m], dp[m], dot);
      }
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int j = lane + 32 * m;
      if (j < N) dS[i * LDN + j] = p[m] * (dp[m] - dot) * scale;
    }
  }
  __syncthreads();
  for (int i = warp; i < N; i += 8) {
    float* out = dqkv + (size_t)(b * N + i) * 1536 + h * 128;
    for (int c = lane; c < 128; c += 32) {
      float dq = 0.f, dk = 0.f, dv = 0.f;
      for (int j = 0; j < N; ++j) {
        dq = fmaf(dS[i * LDN + j], Ks[j * LD + c], dq);
        dk = fmaf(dS[j * LDN + i], Qs[j * LD + c], dk);
        dv = fmaf(Pd[j * LDN + i], Gs[j * LD + c], dv);
      }
      out[c] = dq;
      out[512 + c] = dk;
      out[1024 + c] = dv;
    }
  }
}

// t-embedding gradient per sequence: dtemb[b] = (sum over the sequence's tokens of dh0) . W_first[:, 189:317]
__global__ void train_dtemb_kernel(const float* __restrict__ dh0, int frames, const float* __restrict__ w_first, float* __restrict__ dtemb) {
  __shared__ float g[512];
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < 512; c += blockDim.x) {
    float a = 0.f;
    for (int n = 0; n < frames; ++n) a += dh0[(size_t)(b * frames + n) * 512 + c];
    g[c] = a;
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    float a = 0.f;
    for (int c = 0; c < 512; ++c) a = fmaf(g[c], w_first[(size_t)c * 702 + 189 + threadIdx.x], a);
    dtemb[b * 128 + threadIdx.x] = a;
  }
}

// time-MLP backward, stage 1 (thread per sequence and hidden unit): du1 = (dtemb W2) * silu'(u1)
__global__ void train_time_du_kernel(const float* __restrict__ dtemb, const float* __restrict__ u1, const float* __restrict__ w2, int B,
                                     float* __restrict__ du1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 128) return;
  const int b = i / 128, k = i % 128;
  float a = 0.f;
  for (int o = 0; o < 128; ++o) a = fmaf(dtemb[b * 128 + o], w2[o * 128 + k], a);
  const float u = u1[i], sg = 1.0f / (1.0f + expf(-u));
  du1[i] = a * sg * (1.0f + u * (1.0f - sg));
}
// stage 2 (thread per weight): dW[o][k] = sum over sequences (in order) of dy[b][o] x[b][k], x = silu(u1) (which = 1) or the
// sinusoidal features of t (which = 0); db[o] = sum of dy[b][o] from the threads with k == 0
__global__ void train_time_dw_kernel(const float* __restrict__ dy, const float* __restrict__ u1, const int* __restrict__ t, int B, int K,
                                     int which, float* __restrict__ dw, float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 128 * K) return;
  const int o = i / K, k = i % K;
  const float freq = expf(-logf(10000.0f) * (float)(k & 127) / 128.0f);
  float a = 0.f, bsum = 0.f;
  for (int b = 0; b < B; ++b) {
    float x;
    if (which) {
      const float u = u1[b * 128 + k];
      x = u / (1.0f + expf(-u));
    } else {
      const float arg = (float)t[b] * freq;
      x = k < 128 ? cosf(arg) : sinf(arg);
    }
    const float g = dy[b * 128 + o];
    a = fmaf(g, x, a);
    bsum += g;
  }
  dw[i] = a;
  if (k == 0) db[o] = bsum;
}

// dL/dx of the harmonic feed columns (Denoiser.forward's backward), thread per (token, pose dimension i):
// dx[i] = dfeed[180 + i] + sum_k 2^k (cos(2^k x_i) dfeed[10 i + k] - sin(2^k x_i) dfeed[90 + 10 i + k]), with sin and cos read back
// from the saved feed row; dfeed [S, 192] holds dL/dfeed of columns 0..188
__global__ void train_dx_kernel(const float* __restrict__ feed, const float* __restrict__ dfeed, int S, float* __restrict__ dx) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= S * 9) return;
  const int s = e / 9, i = e - s * 9;
  const float* f = feed + (size_t)s * kFeedPad;
  const float* g = dfeed + (size_t)s * 192;
  float a = 0.f;
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const int c = 10 * i + k;
    a = fmaf((float)(1 << k), fmaf(f[90 + c], g[c], -f[c] * g[90 + c]), a);
  }
  dx[e] = g[180 + i] + a;
}

}  // namespace
