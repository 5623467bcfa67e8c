// What the two training paths share (csrc/api_train.cu: denoiser, csrc/api_vit_train.cu: image backbone): how a linear layer is
// differentiated on the tensor-core engine, the LayerNorm row arithmetic, the deterministic column reductions, the workspace
// cursor and the launch bookkeeping.
// Gradients are reproducible because of three rules that the code below applies for both paths: no GEMM takes the split-K
// regime, so every output element is one CTA's fixed-order dot product; token counts are zero-padded to a multiple of 32
// before they become a GEMM's K; every reduction over tokens is split into kRedChunks token chunks whose partials are added in
// chunk order (no floating-point atomics).
// The kernels sit in an anonymous namespace so that each including translation unit owns its copy.
#pragma once
#include <cstdint>
#include <utility>

#include "common.cuh"
#include "context.cuh"
#include "tc_linear.cuh"

namespace pdb {

constexpr int kRedChunks = 128;  // token chunks of the deterministic column reductions

}  // namespace pdb

namespace {
using namespace pdb;

// ---- LayerNorm of one row held by one warp, P = C / 32 values per lane (column lane + 32 i in v[i]), biased variance ----------
template <int P>
__device__ __forceinline__ void ln_row_stats(const float (&v)[P], float eps, float& mean, float& rstd) {
  constexpr int C = 32 * P;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < P; ++i) sum += v[i];
  mean = warp_sum(sum) * (1.0f / C);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < P; ++i) sq += (v[i] - mean) * (v[i] - mean);
  rstd = 1.0f / sqrtf(warp_sum(sq) * (1.0f / C) + eps);
}
// Row backward, dx = rstd (g - mean(g) - xhat mean(g xhat)) with g = dy * gamma, in two steps: the two row means, then one
// element.  A caller that adds dx to a residual writes `res + ln_row_dx(...)`, which compiles to the fused multiply-add it would
// be if the expression stood there.
template <int P>
__device__ __forceinline__ void ln_row_bwd_means(const float (&xh)[P], const float (&g)[P], float& mg, float& mgx) {
  constexpr int C = 32 * P;
  float sg = 0.f, sgx = 0.f;
#pragma unroll
  for (int i = 0; i < P; ++i) {
    sg += g[i];
    sgx += g[i] * xh[i];
  }
  mg = warp_sum(sg) * (1.0f / C);
  mgx = warp_sum(sgx) * (1.0f / C);
}
__device__ __forceinline__ float ln_row_dx(float xh, float g, float mg, float mgx, float rstd) { return rstd * (g - mg - xh * mgx); }

// LayerNorm over C columns, one warp per row; stats[row] = {mean, rstd}
template <int C>
__global__ void train_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ bta, int S,
                                    float eps, float* __restrict__ y, float* __restrict__ stats) {
  constexpr int P = C / 32;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= S) return;
  const float* xr = x + (size_t)row * C;
  float v[P], mean, rstd;
#pragma unroll
  for (int i = 0; i < P; ++i) v[i] = xr[lane + 32 * i];
  ln_row_stats(v, eps, mean, rstd);
#pragma unroll
  for (int i = 0; i < P; ++i) {
    const int c = lane + 32 * i;
    y[(size_t)row * C + c] = (v[i] - mean) * rstd * g[c] + bta[c];
  }
  if (lane == 0) {
    stats[2 * row] = mean;
    stats[2 * row + 1] = rstd;
  }
}

// LayerNorm backward, warp per row: out = (res ? res : 0) + dx; prod = dy * xhat (its column sums are the gamma gradient)
template <int C>
__global__ void train_ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ stats,
                                    const float* __restrict__ gamma, const float* res, int S, float* out, float* __restrict__ prod) {
  constexpr int P = C / 32;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= S) return;
  const float mean = stats[2 * row], rstd = stats[2 * row + 1];
  float xh[P], g[P], mg, mgx;
#pragma unroll
  for (int i = 0; i < P; ++i) {
    const int c = lane + 32 * i;
    const float d = dy[(size_t)row * C + c];
    xh[i] = (x[(size_t)row * C + c] - mean) * rstd;
    g[i] = d * gamma[c];
    prod[(size_t)row * C + c] = d * xh[i];
  }
  ln_row_bwd_means(xh, g, mg, mgx);
#pragma unroll
  for (int i = 0; i < P; ++i) {
    const int c = lane + 32 * i;
    const float dx = ln_row_dx(xh[i], g[i], mg, mgx, rstd);
    out[(size_t)row * C + c] = res ? res[(size_t)row * C + c] + dx : dx;
  }
}

// out[C, Rp] = in[R, C]^T, rows R..Rp-1 of the result zero (token padding of the weight-gradient GEMMs)
__global__ void train_transpose_kernel(const float* __restrict__ in, int R, int C, int Rp, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int k = threadIdx.y; k < 32; k += blockDim.y) {
    const int r = r0 + k, c = c0 + threadIdx.x;
    tile[k][threadIdx.x] = (r < R && c < C) ? in[(size_t)r * C + c] : 0.f;
  }
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += blockDim.y) {
    const int c = c0 + k, r = r0 + threadIdx.x;
    if (c < C && r < Rp) out[(size_t)c * Rp + r] = tile[threadIdx.x][k];
  }
}

// copy rows x cols of src (leading dimension lds) into dst (leading dimension ldd), columns cols..ldd-1 of dst zero
__global__ void train_copy_cols_kernel(const float* __restrict__ src, int lds, int rows, int cols, float* __restrict__ dst, int ldd) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * ldd) return;
  const int r = (int)(i / ldd), c = (int)(i % ldd);
  dst[i] = c < cols ? src[(size_t)r * lds + c] : 0.f;
}

// deterministic column sums, stage 1: partial[chunk][c] = sum over the chunk's rows of A[row][c] (rows in order)
__global__ void train_colsum_partial_kernel(const float* __restrict__ A, int S, int C, float* __restrict__ partial) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, chunk = blockIdx.y;
  if (c >= C) return;
  const int per = (S + kRedChunks - 1) / kRedChunks, s0 = chunk * per, s1 = min(S, s0 + per);
  float acc = 0.f;
  for (int s = s0; s < s1; ++s) acc += A[(size_t)s * C + c];
  partial[(size_t)chunk * C + c] = acc;
}
// stage 2: out[c] = sum over chunks in chunk order
__global__ void train_chunk_sum_kernel(const float* __restrict__ partial, int chunks, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (int k = 0; k < chunks; ++k) acc += partial[(size_t)k * C + c];
  out[c] = acc;
}

// ---- host side ---------------------------------------------------------------------------------------------------------------
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

unsigned blocks(long long n, int per = 256) { return (unsigned)((n + per - 1) / per); }

// Offsets into a training workspace, in floats: a 64-float header, then blocks that each start 64-float aligned
struct WorkspaceCursor {
  size_t at = 64;
  size_t take(size_t n) {
    const size_t o = at;
    at += (n + 63) / 64 * 64;
    return o;
  }
};

// Every kernel the training entry points enqueue themselves goes through here, so that pdb_launch_count is the number of
// kernels enqueued (the GEMMs count themselves in enqueue_tc_linear).  A plain <<<>>> launch: no launch attributes.
template <typename... Params, typename... Args>
void train_launch(Context* ctx, cudaStream_t st, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
  ctx->launches += 1;
}

// Y[S, O] = relu?(X[S, K] W[O, K]^T + bias) + residual
int train_gemm(Context* ctx, const float* X, const float* W, const float* bias, const float* residual, float* Y, int S, int O, int K,
               int relu, cudaStream_t st) {
  TcEpilogue E = {};
  E.bias = bias;
  E.residual = residual;
  E.ldr = O;
  E.Y = Y;
  E.ldy = O;
  E.S = S;
  E.O = O;
  E.K = K;
  E.relu = relu;
  E.allow_small = 0;  // no split-K: every output element is one CTA's dot product in k order
  return enqueue_tc_linear(ctx, X, W, E, st);
}

// The three gradients of Y[S, O] = X[S, K] W[O, K]^T + b from dY.  Borrows the caller's scratch: T1 holds the largest dY^T
// [O, Sp], T2 the largest X^T [K, Sp], Wt the largest weight, part kRedChunks rows of the widest bias; Sp = S rounded up to 32.
struct LinearGrad {
  Context* ctx;
  int S, Sp;
  float *T1, *T2, *Wt, *part;
  cudaStream_t st;

  // dW[O, K] = dY[S, O]^T X[S, K] over the token-major transposes (zero-padded to Sp tokens)
  int weight(const float* dY, int O, const float* X, int K, float* dW) const {
    transpose(dY, S, O, Sp, T1);
    transpose(X, S, K, Sp, T2);
    return train_gemm(ctx, T1, T2, nullptr, nullptr, dW, O, K, Sp, 0, st);
  }
  // dX[S, K] = dY[S, O] W[O, K] with W transposed to K-major
  int input(const float* dY, const float* W, int O, int K, float* dX) const {
    transpose(W, O, K, O, Wt);
    return train_gemm(ctx, dY, Wt, nullptr, nullptr, dX, S, K, O, 0, st);
  }
  // db[O] = column sums of dY[rows, O]
  void bias(const float* dY, int rows, int O, float* db) const {
    train_launch(ctx, st, train_colsum_partial_kernel, dim3((O + 255) / 256, kRedChunks), 256, 0, dY, rows, O, part);
    train_launch(ctx, st, train_chunk_sum_kernel, (O + 255) / 256, 256, 0, part, kRedChunks, O, db);
  }

 private:
  void transpose(const float* in, int R, int C, int Rp, float* out) const {
    train_launch(ctx, st, train_transpose_kernel, dim3((C + 31) / 32, (Rp + 31) / 32), dim3(32, 8), 0, in, R, C, Rp, out);
  }
};

}  // namespace
