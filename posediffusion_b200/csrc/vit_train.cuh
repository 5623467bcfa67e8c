// Training kernels of the DINO ViT-S/16 backbone (csrc/api_vit_train.cu): what the backward needs beyond the shared pieces of
// csrc/vit.cuh (patchify, attention forward, head) and csrc/train_common.cuh (LayerNorm forward / backward, the linear-layer
// backward, column sums).
// All fp32 CUDA-core code; the projections and their gradients run on the tensor-core linear layer.  Every reduction over tokens
// or images is a fixed-order sum: no floating-point atomics, two runs give bit-identical gradients.
#pragma once
#include "train_common.cuh"
#include "vit.cuh"

namespace {
using namespace pdb;

// ---- exact (erf) GELU, recomputed in the backward from the saved fc1 pre-activation ----
__global__ void vit_gelu_fwd_kernel(const float* __restrict__ u, float* __restrict__ y, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = u[i];
  y[i] = 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
}
// g *= gelu'(u) = Phi(u) + u phi(u)
__global__ void vit_gelu_bwd_kernel(float* __restrict__ g, const float* __restrict__ u, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = u[i];
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * expf(-0.5f * x * x);
  g[i] *= cdf + x * pdf;
}

// ---- position table of one resampled scale: out[0] = pos[0], out[1 + p] = sum_k weight[16 p + k] * pos[1 + cell[16 p + k]] ----
// Products and sums rounded separately, in tap order: the same values resample_pos computes on the host.
__global__ void vit_pos_apply_kernel(const float* __restrict__ pos, const int* __restrict__ cell, const float* __restrict__ weight,
                                     int tokens, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= tokens * kVitDim) return;
  const int tok = idx / kVitDim, c = idx - tok * kVitDim;
  float acc = pos[c];
  if (tok > 0) {
    acc = 0.f;
    for (int k = 0; k < kVitPosTaps; ++k) {
      const int t = (tok - 1) * kVitPosTaps + k;
      acc = __fadd_rn(acc, __fmul_rn(weight[t], pos[(size_t)(1 + cell[t]) * kVitDim + c]));
    }
  }
  out[idx] = acc;
}

// ---- head backward: z = mean over scales of LayerNorm(class row), so every scale's class row receives dz / n_scales through the
// final norm.  One warp per (scale, image): dX class row, and the rows whose column sums are the norm's gamma / beta gradients.
__global__ void vit_head_bwd_kernel(const float* __restrict__ X, VitHeadArgs a, const float* __restrict__ gamma,
                                    const float* __restrict__ gz, int n_images, float* __restrict__ dX, float* __restrict__ prod,
                                    float* __restrict__ dy_rows) {
  const int item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (item >= a.n_scales * n_images) return;
  const int s = item / n_images, n = item - s * n_images;
  const size_t row = (size_t)(a.row0[s] + n * a.tokens[s]);
  constexpr int P = kVitDim / 32;
  float v[P], g[P], m, rstd, mg, mgx;
#pragma unroll
  for (int i = 0; i < P; ++i) v[i] = X[row * kVitDim + lane + 32 * i];
  ln_row_stats(v, kVitLnEps, m, rstd);
#pragma unroll
  for (int i = 0; i < P; ++i) {
    const int c = lane + 32 * i;
    const float dy = gz[(size_t)n * kVitDim + c] / (float)a.n_scales;
    v[i] = (v[i] - m) * rstd;
    g[i] = dy * gamma[c];
    prod[(size_t)item * kVitDim + c] = dy * v[i];
    dy_rows[(size_t)item * kVitDim + c] = dy;
  }
  ln_row_bwd_means(v, g, mg, mgx);
#pragma unroll
  for (int i = 0; i < P; ++i) dX[row * kVitDim + lane + 32 * i] = ln_row_dx(v[i], g[i], mg, mgx, rstd);
}

// ---- attention backward of one (sequence, head), L <= 256 tokens, head width 64, fp32 in shared memory ----
// The probabilities are not stored by the forward; they are recomputed from Q and K.  Two passes over one CTA's shared memory:
//   pass 1 (K, V resident; warp per query row i, lane per key): s = q_i K^T / 8, softmax row, dP = dO_i V^T, delta_i = sum_j P dP,
//           dS = P (dP - delta_i) / 8 -> dQ_i = dS K; the row's log-sum-exp and delta_i are kept for pass 2;
//   pass 2 (Q, dO resident; warp per key row j, lane per query): P and dS of column j from the kept row statistics ->
//           dK_j = dS^T Q, dV_j = P^T dO.
// Rows are padded to 65 words: a warp's 32 rows land in 32 banks.
constexpr int kVitAttBwdLd = 65;
__host__ __device__ inline size_t vit_attn_bwd_smem(int L) {
  return sizeof(float) * ((size_t)2 * L * kVitAttBwdLd + 2 * kVitMaxTokens + 8 * (2 * kVitMaxTokens + 2 * kVitHD));
}
__global__ void __launch_bounds__(256) vit_attn_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ datt, int row0, int L,
                                                           float* __restrict__ dqkv) {
  extern __shared__ float vsm_bwd[];
  constexpr int LD = kVitAttBwdLd;
  float* A = vsm_bwd;
  float* B = A + L * LD;
  float* lse = B + L * LD;
  float* delta = lse + kVitMaxTokens;
  float* wds = delta + kVitMaxTokens;     // [8][256]
  float* wp = wds + 8 * kVitMaxTokens;    // [8][256]
  float* wa = wp + 8 * kVitMaxTokens;     // [8][64]
  float* wb = wa + 8 * kVitHD;            // [8][64]
  const int seq = blockIdx.x / kVitHeads, head = blockIdx.x - seq * kVitHeads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t base = (size_t)(row0 + seq * L);
  const float* q0 = qkv + base * (3 * kVitDim) + head * kVitHD;
  const float* g0 = datt + base * kVitDim + head * kVitHD;
  float* o0 = dqkv + base * (3 * kVitDim) + head * kVitHD;
  const float scale = 0.125f;  // head_dim ** -0.5
  float* ds_row = wds + warp * kVitMaxTokens;
  float* p_row = wp + warp * kVitMaxTokens;
  float* ra = wa + warp * kVitHD;
  float* rb = wb + warp * kVitHD;

  for (int idx = threadIdx.x; idx < L * kVitHD; idx += blockDim.x) {
    const int j = idx >> 6, c = idx & 63;
    A[j * LD + c] = q0[(size_t)j * (3 * kVitDim) + kVitDim + c];      // K
    B[j * LD + c] = q0[(size_t)j * (3 * kVitDim) + 2 * kVitDim + c];  // V
  }
  __syncthreads();
  for (int i = warp; i < L; i += 8) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      ra[lane + 32 * h] = q0[(size_t)i * (3 * kVitDim) + lane + 32 * h] * scale;
      rb[lane + 32 * h] = g0[(size_t)i * kVitDim + lane + 32 * h];
    }
    __syncwarp();
    float s[8], dp[8], mx = -INFINITY;
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      const int j = lane + 32 * m;
      s[m] = -INFINITY;
      dp[m] = 0.f;
      if (j < L) {
        float a = 0.f, b = 0.f;
        for (int c = 0; c < kVitHD; ++c) {
          a = fmaf(ra[c], A[j * LD + c], a);
          b = fmaf(rb[c], B[j * LD + c], b);
        }
        s[m] = a;
        dp[m] = b;
      }
      mx = fmaxf(mx, s[m]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      s[m] = (lane + 32 * m < L) ? expf(s[m] - mx) : 0.f;
      sum += s[m];
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    float dot = 0.f;
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      s[m] *= inv;
      dot = fmaf(s[m], dp[m], dot);
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      const int j = lane + 32 * m;
      if (j < L) ds_row[j] = s[m] * (dp[m] - dot) * scale;
    }
    if (lane == 0) {
      lse[i] = mx + logf(sum);
      delta[i] = dot;
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = lane + 32 * h;
      float acc = 0.f;
      for (int j = 0; j < L; ++j) acc = fmaf(ds_row[j], A[j * LD + c], acc);
      o0[(size_t)i * (3 * kVitDim) + c] = acc;
    }
    __syncwarp();
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < L * kVitHD; idx += blockDim.x) {
    const int j = idx >> 6, c = idx & 63;
    A[j * LD + c] = q0[(size_t)j * (3 * kVitDim) + c];  // Q
    B[j * LD + c] = g0[(size_t)j * kVitDim + c];        // dO
  }
  __syncthreads();
  for (int j = warp; j < L; j += 8) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      ra[lane + 32 * h] = q0[(size_t)j * (3 * kVitDim) + kVitDim + lane + 32 * h];      // K_j
      rb[lane + 32 * h] = q0[(size_t)j * (3 * kVitDim) + 2 * kVitDim + lane + 32 * h];  // V_j
    }
    __syncwarp();
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      const int i = lane + 32 * m;
      if (i < L) {
        float a = 0.f, b = 0.f;
        for (int c = 0; c < kVitHD; ++c) {
          a = fmaf(A[i * LD + c], ra[c], a);
          b = fmaf(B[i * LD + c], rb[c], b);
        }
        const float p = expf(a * scale - lse[i]);
        p_row[i] = p;
        ds_row[i] = p * (b - delta[i]) * scale;
      }
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = lane + 32 * h;
      float dk = 0.f, dv = 0.f;
      for (int i = 0; i < L; ++i) {
        dk = fmaf(ds_row[i], A[i * LD + c], dk);
        dv = fmaf(p_row[i], B[i * LD + c], dv);
      }
      o0[(size_t)j * (3 * kVitDim) + kVitDim + c] = dk;
      o0[(size_t)j * (3 * kVitDim) + 2 * kVitDim + c] = dv;
    }
    __syncwarp();
  }
}

// ---- position embedding, class token and patch bias gradients ----
// stage 1: sum[tok][c] = sum over the scale's images (in order) of dX0[row0 + n * tokens + tok][c]
__global__ void vit_pos_sum_kernel(const float* __restrict__ dX0, int row0, int tokens, int n_images, float* __restrict__ sum) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= tokens * kVitDim) return;
  const float* p = dX0 + (size_t)row0 * kVitDim + idx;
  float acc = 0.f;
  for (int n = 0; n < n_images; ++n) acc += p[(size_t)n * tokens * kVitDim];
  sum[idx] = acc;
}
struct VitPosGradArgs {
  int n_scales;
  int tokens[kVitMaxScales];
  int resampled[kVitMaxScales];       // 0: the scale used the stored table itself
  const float* sum[kVitMaxScales];    // [tokens, 384] from stage 1
  const int* cell[kVitMaxScales];     // taps of R_s (resampled scales)
  const float* weight[kVitMaxScales];
};
// stage 2, thread per (stored position i, column): d pos_embed[i] = sum over scales (in order) of R_s^T applied to that scale's
// sums, the adjoint gathered per stored cell in (patch, tap) order.  The class position i = 0 also gives d cls_token, and the
// same threads add up the patch rows into d patch bias (the class rows never saw the bias).
__global__ void vit_pos_grad_kernel(VitPosGradArgs a, float* __restrict__ dpos, float* __restrict__ dcls, float* __restrict__ dbias) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (1 + kVitGrid0 * kVitGrid0) * kVitDim) return;
  const int i = idx / kVitDim, c = idx - i * kVitDim;
  float acc = 0.f;
  if (i == 0) {
    float bias = 0.f;
    for (int s = 0; s < a.n_scales; ++s) {
      acc += a.sum[s][c];
      for (int tok = 1; tok < a.tokens[s]; ++tok) bias += a.sum[s][(size_t)tok * kVitDim + c];
    }
    dcls[c] = acc;
    dbias[c] = bias;
  } else {
    for (int s = 0; s < a.n_scales; ++s) {
      if (!a.resampled[s]) {
        acc += a.sum[s][(size_t)i * kVitDim + c];
        continue;
      }
      const int taps = (a.tokens[s] - 1) * kVitPosTaps;
      for (int t = 0; t < taps; ++t)
        if (a.cell[s][t] == i - 1) acc = fmaf(a.weight[s][t], a.sum[s][(size_t)(1 + t / kVitPosTaps) * kVitDim + c], acc);
    }
  }
  dpos[idx] = acc;
}

}  // namespace
