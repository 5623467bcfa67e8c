// Training entry points of the denoiser: GaussianDiffusion.p_losses forward with every activation the backward needs saved in a
// caller-owned workspace, the backward into 108 parameter gradients, camera_to_pose_encoding, and the host image of the dropout
// masks.  Projections run through enqueue_tc_linear (TF32 products, fp32 accumulate) without its split-K regime, so every output
// element is one CTA's fixed-order dot product; all other reductions are chunked fixed-order sums (csrc/train.cuh).
#include <cmath>
#include <cstring>

#include "context.cuh"
#include "denoiser.cuh"
#include "tc_linear.cuh"
#include "train.cuh"

using namespace pdb;

namespace {

constexpr int kMagic = 0x7d1a1e01;

// Workspace: a 64-float header, the saved activations, then the backward's scratch.  Offsets in floats, each 64-float aligned.
struct TrainLayout {
  int B, N, S, Sp;
  size_t t, feed, u1, temb, hin[kLayers + 1], a1[kLayers], st1[kLayers], qkv[kLayers], P[kLayers], att[kLayers], hmid[kLayers],
      a2[kLayers], st2[kLayers], fd[kLayers], u, stu, r, diff;
  size_t D0, D1, G1, G2, T1, T2, Wt, part, Wpad, dWf, deps, dtemb, du1;
  size_t total;
  TrainLayout(int batch, int frames) : B(batch), N(frames), S(batch * frames), Sp((batch * frames + 31) / 32 * 32) {
    size_t at = 64;
    auto take = [&](size_t n) { size_t o = at; at += (n + 63) / 64 * 64; return o; };
    const size_t s = (size_t)S;
    t = take(B);
    feed = take(s * kFeedPad);
    u1 = take((size_t)B * 128);
    temb = take((size_t)B * 128);
    for (int l = 0; l <= kLayers; ++l) hin[l] = take(s * kDM);
    for (int l = 0; l < kLayers; ++l) {
      a1[l] = take(s * kDM); st1[l] = take(2 * s); qkv[l] = take(s * 3 * kDM); P[l] = take((size_t)B * kHeads * N * N);
      att[l] = take(s * kDM); hmid[l] = take(s * kDM); a2[l] = take(s * kDM); st2[l] = take(2 * s); fd[l] = take(s * kFF);
    }
    u = take(s * kHid); stu = take(2 * s); r = take(s * kHid); diff = take(s * 9);
    D0 = take(s * kDM); D1 = take(s * kDM); G1 = take(s * 3 * kDM); G2 = take(s * kFF);
    T1 = take((size_t)3 * kDM * Sp); T2 = take((size_t)kFF * Sp); Wt = take((size_t)3 * kDM * kDM);
    part = take((size_t)kRedChunks * 3 * kDM); Wpad = take((size_t)kDM * kFeedPad); dWf = take((size_t)kDM * kFeedPad);
    deps = take(s * 9); dtemb = take((size_t)B * 128); du1 = take((size_t)B * 128);
    total = at;
  }
};

struct TrainHeader {
  int32_t magic, batch, frames, loss_type;
  uint32_t threshold, seed_lo, seed_hi;
  float scale;
  int32_t bad_t;  // set when a timestep lies outside [0, kT): the backward then refuses the workspace
};
// header + the timesteps the kernels index the schedule with, clamped into [0, kT) so that no kernel reads past it; an
// out-of-range input is flagged in the header instead (reading it back here would synchronise the forward)
__global__ void train_header_kernel(TrainHeader h, int* __restrict__ dst, const int* __restrict__ t, int* __restrict__ t_copy) {
  TrainHeader* hd = reinterpret_cast<TrainHeader*>(dst);
  if (threadIdx.x == 0) *hd = h;
  __syncthreads();
  for (int b = threadIdx.x; b < h.batch; b += blockDim.x) {
    const int v = t[b];
    t_copy[b] = min(max(v, 0), kT - 1);
    if (v < 0 || v >= kT) atomicExch(&hd->bad_t, 1);
  }
}

TrainSched train_schedule() {
  TrainSched sc;
  const int n = kT;
  const double b1 = 1e-4, bT = 0.1, step = (bT - b1) / (double)(n - 1);
  double prod = 1.0;
  for (int i = 0; i < n; ++i) {
    const double beta = (i < n / 2) ? b1 + step * i : bT - step * (n - 1 - i);  // torch.linspace fills from both ends
    prod *= (1.0 - beta);
    sc.c[i][0] = (float)std::sqrt(prod);
    sc.c[i][1] = (float)std::sqrt(1.0 - prod);
    sc.c[i][2] = (float)std::sqrt(1.0 / prod);
    sc.c[i][3] = (float)std::sqrt(1.0 / prod - 1.0);
  }
  return sc;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_params(Context* ctx, const float* const* params) {
  if (!params) return ctx->fail(PDB_ERR_INVALID, "params is null");
  for (int i = 0; i < PDB_NUM_WEIGHT_TENSORS; ++i) {
    if (!params[i]) return ctx->fail(PDB_ERR_INVALID, "parameter %d is null", i);
    if (!aligned16(params[i])) return ctx->fail(PDB_ERR_INVALID, "parameter %d is not 16-byte aligned", i);
  }
  return PDB_OK;
}

int gemm(Context* ctx, const float* X, const float* W, const float* bias, float* Y, int S, int O, int K, int relu, cudaStream_t st) {
  TcEpilogue E = {};
  E.bias = bias;
  E.Y = Y;
  E.ldy = O;
  E.S = S;
  E.O = O;
  E.K = K;
  E.relu = relu;
  E.allow_small = 0;  // no split-K: every output element is one CTA's dot product in k order
  return enqueue_tc_linear(ctx, X, W, E, st);
}

void transpose(const float* in, int R, int C, int Rp, float* out, cudaStream_t st) {
  train_transpose_kernel<<<dim3((C + 31) / 32, (Rp + 31) / 32), dim3(32, 8), 0, st>>>(in, R, C, Rp, out);
}

void colsum(const float* A, int S, int C, float* partial, float* out, cudaStream_t st) {
  train_colsum_partial_kernel<<<dim3((C + 255) / 256, kRedChunks), 256, 0, st>>>(A, S, C, partial);
  train_chunk_sum_kernel<<<(C + 255) / 256, 256, 0, st>>>(partial, kRedChunks, C, out);
}

size_t attn_fwd_smem(int N) { return sizeof(float) * ((size_t)2 * N * 129 + 8 * 128 + 8 * 64); }
size_t attn_bwd_smem(int N) { return sizeof(float) * ((size_t)4 * N * 129 + (size_t)2 * N * (N + 1)); }

int set_attn_smem(Context* ctx) {
  static bool done[64] = {};
  int dev = ctx->device;
  if (dev >= 0 && dev < 64 && !done[dev]) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(train_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_fwd_smem(kTrainMaxFrames)));
    PDB_CUDA(ctx, cudaFuncSetAttribute(train_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_bwd_smem(kTrainMaxFrames)));
    done[dev] = true;
  }
  return PDB_OK;
}

DropCfg drop_cfg(uint32_t threshold, float scale, uint64_t seed) {
  DropCfg d;
  d.seed = seed;
  d.threshold = threshold;
  d.scale = scale;
  return d;
}

unsigned blocks(long long n, int per = 256) { return (unsigned)((n + per - 1) / per); }

}  // namespace

extern "C" int64_t pdb_train_workspace_bytes(int32_t batch, int32_t frames) {
  if (batch < 1 || frames < 1 || frames > kTrainMaxFrames) return 0;
  return (int64_t)(TrainLayout(batch, frames).total * sizeof(float));
}

extern "C" int pdb_train_forward(pdb_context* c, const float* const* params, const float* x_start, const int32_t* t, const float* noise,
                                 const float* z, int32_t batch, int32_t frames, float dropout_p, uint64_t seed, int32_t loss_type,
                                 void* workspace, float* loss, float* x_t, float* x0, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (int rc = check_params(ctx, params)) return rc;
  if (!x_start || !t || !noise || !z || !workspace || !loss || !x_t || !x0) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (!aligned16(workspace)) return ctx->fail(PDB_ERR_INVALID, "workspace is not 16-byte aligned");
  if (batch < 1 || frames < 1) return ctx->fail(PDB_ERR_INVALID, "batch %d, frames %d", batch, frames);
  if (frames > kTrainMaxFrames) return ctx->fail(PDB_ERR_LIMIT, "training supports at most %d frames per sequence, got %d", kTrainMaxFrames, frames);
  if (!(dropout_p >= 0.f && dropout_p < 1.f)) return ctx->fail(PDB_ERR_INVALID, "dropout probability %g outside [0, 1)", (double)dropout_p);
  if (loss_type != 0 && loss_type != 1) return ctx->fail(PDB_ERR_INVALID, "loss_type %d (0 = l1, 1 = l2)", loss_type);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (int rc = set_attn_smem(ctx)) return rc;
  const TrainLayout L(batch, frames);
  float* ws = static_cast<float*>(workspace);
  const int S = L.S, B = batch, N = frames;
  const TrainSched sc = train_schedule();
  const DropCfg d = drop_cfg(dropout_threshold(dropout_p), 1.0f / (1.0f - dropout_p), seed);
  int* tsv = reinterpret_cast<int*>(ws + L.t);
  TrainHeader hdr = {kMagic, batch, frames, loss_type, d.threshold, (uint32_t)seed, (uint32_t)(seed >> 32), d.scale, 0};
  train_header_kernel<<<1, 128, 0, st>>>(hdr, reinterpret_cast<int*>(ws), t, tsv);
  auto W = [&](int i) { return params[i]; };
  // feed
  train_time_mlp_kernel<<<B, 128, 0, st>>>(tsv, W(0), W(1), W(2), W(3), ws + L.u1, ws + L.temb);
  train_feed_kernel<<<S, 256, 0, st>>>(sc, x_start, noise, tsv, ws + L.temb, z, N, S, x_t, ws + L.feed);
  train_copy_cols_kernel<<<blocks((long long)kDM * kFeedPad), 256, 0, st>>>(W(4), kFirstIn, kDM, kFirstIn, ws + L.Wpad, kFeedPad);
  if (int rc = gemm(ctx, ws + L.feed, ws + L.Wpad, W(5), ws + L.hin[0], S, kDM, kFeedPad, 0, st)) return rc;
  const long long nd = (long long)S * kDM, nf = (long long)S * kFF;
  for (int l = 0; l < kLayers; ++l) {
    const int b = 6 + 12 * l;
    train_ln_fwd_kernel<kDM><<<blocks(S, 8), 256, 0, st>>>(ws + L.hin[l], W(b + 8), W(b + 9), S, kLnEps, ws + L.a1[l], ws + L.st1[l]);
    if (int rc = gemm(ctx, ws + L.a1[l], W(b + 0), W(b + 1), ws + L.qkv[l], S, 3 * kDM, kDM, 0, st)) return rc;
    train_attn_fwd_kernel<<<B * kHeads, 256, attn_fwd_smem(N), st>>>(ws + L.qkv[l], N, d, l, ws + L.P[l], ws + L.att[l]);
    if (int rc = gemm(ctx, ws + L.att[l], W(b + 2), W(b + 3), ws + L.G1, S, kDM, kDM, 0, st)) return rc;
    train_dropout_kernel<<<blocks(nd), 256, 0, st>>>(ws + L.G1, ws + L.hin[l], nullptr, ws + L.hmid[l], nd, d, l, kSiteOut);
    train_ln_fwd_kernel<kDM><<<blocks(S, 8), 256, 0, st>>>(ws + L.hmid[l], W(b + 10), W(b + 11), S, kLnEps, ws + L.a2[l], ws + L.st2[l]);
    if (int rc = gemm(ctx, ws + L.a2[l], W(b + 4), W(b + 5), ws + L.fd[l], S, kFF, kDM, 1, st)) return rc;
    train_dropout_kernel<<<blocks(nf), 256, 0, st>>>(ws + L.fd[l], nullptr, nullptr, ws + L.fd[l], nf, d, l, kSiteRelu);
    if (int rc = gemm(ctx, ws + L.fd[l], W(b + 6), W(b + 7), ws + L.G1, S, kDM, kFF, 0, st)) return rc;
    train_dropout_kernel<<<blocks(nd), 256, 0, st>>>(ws + L.G1, ws + L.hmid[l], nullptr, ws + L.hin[l + 1], nd, d, l, kSiteFF2);
  }
  const int tb = 6 + 12 * kLayers;
  if (int rc = gemm(ctx, ws + L.hin[kLayers], W(tb), W(tb + 1), ws + L.u, S, kHid, kDM, 0, st)) return rc;
  train_tail_fwd_kernel<<<blocks(S, 8), 256, 0, st>>>(sc, ws + L.u, W(tb + 2), W(tb + 3), W(tb + 4), W(tb + 5), tsv, x_t, noise, N, S,
                                                      loss_type, ws + L.stu, ws + L.r, ws + L.diff, loss, x0);
  ctx->launches += 6 + kLayers * 10 + 2;
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

extern "C" int pdb_train_backward(pdb_context* c, const float* const* params, void* workspace, const float* grad_loss, const float* grad_x0,
                                  float* const* grads, void* stream) {
  return pdb_train_backward_z(c, params, workspace, grad_loss, grad_x0, grads, nullptr, stream);
}

extern "C" int pdb_train_backward_z(pdb_context* c, const float* const* params, void* workspace, const float* grad_loss,
                                    const float* grad_x0, float* const* grads, float* grad_z, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (int rc = check_params(ctx, params)) return rc;
  if (!workspace || !grads) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (grad_z && !aligned16(grad_z)) return ctx->fail(PDB_ERR_INVALID, "grad_z is not 16-byte aligned");
  for (int i = 0; i < PDB_NUM_WEIGHT_TENSORS; ++i)
    if (!grads[i] || !aligned16(grads[i])) return ctx->fail(PDB_ERR_INVALID, "gradient %d is null or not 16-byte aligned", i);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (int rc = set_attn_smem(ctx)) return rc;
  float* ws = static_cast<float*>(workspace);
  TrainHeader hdr;
  PDB_CUDA(ctx, cudaMemcpyAsync(&hdr, ws, sizeof(hdr), cudaMemcpyDeviceToHost, st));
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  if (hdr.magic != kMagic || hdr.batch < 1 || hdr.frames < 1 || hdr.frames > kTrainMaxFrames)
    return ctx->fail(PDB_ERR_STATE, "workspace does not hold a training forward");
  if (hdr.bad_t) return ctx->fail(PDB_ERR_INVALID, "the forward was given a timestep outside [0, %d)", kT);
  const TrainLayout L(hdr.batch, hdr.frames);
  const int S = L.S, Sp = L.Sp, B = hdr.batch, N = hdr.frames;
  const TrainSched sc = train_schedule();
  const DropCfg d = drop_cfg(hdr.threshold, hdr.scale, (uint64_t)hdr.seed_lo | ((uint64_t)hdr.seed_hi << 32));
  const int* tsv = reinterpret_cast<const int*>(ws + L.t);
  auto W = [&](int i) { return params[i]; };
  auto G = [&](int i) { return grads[i]; };
  float *D0 = ws + L.D0, *D1 = ws + L.D1, *G1 = ws + L.G1, *G2 = ws + L.G2, *T1 = ws + L.T1, *T2 = ws + L.T2, *Wt = ws + L.Wt;
  float* part = ws + L.part;
  // dW[O, K] = dY[S, O]^T X[S, K] over the token-major transposes (zero-padded to Sp tokens)
  auto weight_grad = [&](const float* dY, int O, const float* X, int K, float* dW) {
    transpose(dY, S, O, Sp, T1, st);
    transpose(X, S, K, Sp, T2, st);
    return gemm(ctx, T1, T2, nullptr, dW, O, K, Sp, 0, st);
  };
  // dX[S, K] = dY[S, O] W[O, K] with W transposed to K-major
  auto input_grad = [&](const float* dY, const float* Wm, int O, int K, float* dX) {
    transpose(Wm, O, K, O, Wt, st);
    return gemm(ctx, dY, Wt, nullptr, dX, S, K, O, 0, st);
  };
  const long long nd = (long long)S * kDM, nf = (long long)S * kFF;
  // ---- tail ----
  const int tb = 6 + 12 * kLayers;
  float* dau = G2;  // [S, 128]
  train_tail_bwd_kernel<<<blocks(S, 8), 256, 0, st>>>(sc, ws + L.diff, grad_loss, grad_x0, tsv, N, S, hdr.loss_type, W(tb + 4), ws + L.r,
                                                      ws + L.deps, dau);
  train_w3_partial_kernel<<<kRedChunks, 128, 0, st>>>(ws + L.deps, ws + L.r, S, part);
  train_chunk_sum_kernel<<<blocks(9 * 128), 256, 0, st>>>(part, kRedChunks, 9 * 128, G(tb + 4));
  colsum(ws + L.deps, S, 9, part, G(tb + 5), st);
  float* du = G1;  // [S, 128]
  train_ln_bwd_kernel<kHid><<<blocks(S, 8), 256, 0, st>>>(dau, ws + L.u, ws + L.stu, W(tb + 2), nullptr, S, du, G2 + (size_t)S * kHid);
  colsum(G2 + (size_t)S * kHid, S, kHid, part, G(tb + 2), st);
  colsum(dau, S, kHid, part, G(tb + 3), st);
  if (int rc = weight_grad(du, kHid, ws + L.hin[kLayers], kDM, G(tb))) return rc;
  colsum(du, S, kHid, part, G(tb + 1), st);
  if (int rc = input_grad(du, W(tb), kHid, kDM, D0)) return rc;
  // ---- trunk, last layer first; D0 = gradient of the layer output ----
  for (int l = kLayers - 1; l >= 0; --l) {
    const int b = 6 + 12 * l;
    float* dy2 = G1;
    train_dropout_kernel<<<blocks(nd), 256, 0, st>>>(D0, nullptr, nullptr, dy2, nd, d, l, kSiteFF2);
    if (int rc = input_grad(dy2, W(b + 6), kDM, kFF, G2)) return rc;  // d fd
    if (int rc = weight_grad(dy2, kDM, ws + L.fd[l], kFF, G(b + 6))) return rc;
    colsum(dy2, S, kDM, part, G(b + 7), st);
    train_dropout_kernel<<<blocks(nf), 256, 0, st>>>(G2, nullptr, ws + L.fd[l], G2, nf, d, l, kSiteRelu);  // d(FF1 output)
    float* da2 = G1;
    if (int rc = input_grad(G2, W(b + 4), kFF, kDM, da2)) return rc;
    if (int rc = weight_grad(G2, kFF, ws + L.a2[l], kDM, G(b + 4))) return rc;
    colsum(G2, S, kFF, part, G(b + 5), st);
    train_ln_bwd_kernel<kDM><<<blocks(S, 8), 256, 0, st>>>(da2, ws + L.hmid[l], ws + L.st2[l], W(b + 10), D0, S, D1, G2);
    colsum(G2, S, kDM, part, G(b + 10), st);
    colsum(da2, S, kDM, part, G(b + 11), st);
    float* dy = G1;
    train_dropout_kernel<<<blocks(nd), 256, 0, st>>>(D1, nullptr, nullptr, dy, nd, d, l, kSiteOut);
    if (int rc = input_grad(dy, W(b + 2), kDM, kDM, G2)) return rc;  // d att
    if (int rc = weight_grad(dy, kDM, ws + L.att[l], kDM, G(b + 2))) return rc;
    colsum(dy, S, kDM, part, G(b + 3), st);
    float* dqkv = G1;
    train_attn_bwd_kernel<<<B * kHeads, 256, attn_bwd_smem(N), st>>>(ws + L.qkv[l], ws + L.P[l], G2, N, d, l, dqkv);
    float* da1 = G2;
    if (int rc = input_grad(dqkv, W(b + 0), 3 * kDM, kDM, da1)) return rc;
    if (int rc = weight_grad(dqkv, 3 * kDM, ws + L.a1[l], kDM, G(b + 0))) return rc;
    colsum(dqkv, S, 3 * kDM, part, G(b + 1), st);
    train_ln_bwd_kernel<kDM><<<blocks(S, 8), 256, 0, st>>>(da1, ws + L.hin[l], ws + L.st1[l], W(b + 8), D1, S, D0, G1);
    colsum(G1, S, kDM, part, G(b + 8), st);
    colsum(da1, S, kDM, part, G(b + 9), st);
  }
  // ---- _first and the time MLP ----
  if (int rc = weight_grad(D0, kDM, ws + L.feed, kFeedPad, ws + L.dWf)) return rc;
  train_copy_cols_kernel<<<blocks((long long)kDM * kFirstIn), 256, 0, st>>>(ws + L.dWf, kFeedPad, kDM, kFirstIn, G(4), kFirstIn);
  colsum(D0, S, kDM, part, G(5), st);
  train_dtemb_kernel<<<B, 256, 0, st>>>(D0, N, W(4), ws + L.dtemb);
  train_time_du_kernel<<<blocks((long long)B * 128), 256, 0, st>>>(ws + L.dtemb, ws + L.u1, W(2), B, ws + L.du1);
  train_time_dw_kernel<<<blocks(128 * 128), 256, 0, st>>>(ws + L.dtemb, ws + L.u1, tsv, B, 128, 1, G(2), G(3));
  train_time_dw_kernel<<<blocks(128 * 256), 256, 0, st>>>(ws + L.du1, ws + L.u1, tsv, B, 256, 0, G(0), G(1));
  ctx->launches += 20 + kLayers * 40;
  if (grad_z) {
    // dz = dh0 . W_first[:, 317:701]: the column block starts at float 317, which TMA cannot address, so it is copied to an
    // aligned [512, 384] buffer (the _first weight-gradient staging area, free by now) and then read K-major like every dX
    float* Wz = ws + L.dWf;
    train_copy_cols_kernel<<<blocks((long long)kDM * kZ), 256, 0, st>>>(W(4) + 317, kFirstIn, kDM, kZ, Wz, kZ);
    if (int rc = input_grad(D0, Wz, kDM, kZ, grad_z)) return rc;
    ctx->launches += 2;
  }
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

// camera_to_pose_encoding, "absT_quaR_logFL" (util/camera_transform.py:108-129) with pytorch3d's matrix_to_quaternion followed by
// standardize_quaternion (real part >= 0): pose = [T | q | log(clamp(focal, min, max)) - bias]
namespace {
__global__ void camera_to_pose_kernel(const float* __restrict__ R, const float* __restrict__ T, const float* __restrict__ F, int count,
                                      float bias, float fmin, float fmax, float* __restrict__ pose) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float* m = R + (size_t)i * 9;
  const float m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7], m22 = m[8];
  const float arg[4] = {1.0f + m00 + m11 + m22, 1.0f + m00 - m11 - m22, 1.0f - m00 + m11 - m22, 1.0f - m00 - m11 + m22};
  float qa[4];
  int best = 0;
  for (int k = 0; k < 4; ++k) {
    qa[k] = arg[k] > 0.f ? sqrtf(arg[k]) : 0.f;
    if (qa[k] > qa[best]) best = k;  // torch.argmax: first maximum
  }
  float q[4];
  switch (best) {
    case 0: q[0] = qa[0] * qa[0]; q[1] = m21 - m12; q[2] = m02 - m20; q[3] = m10 - m01; break;
    case 1: q[0] = m21 - m12; q[1] = qa[1] * qa[1]; q[2] = m10 + m01; q[3] = m02 + m20; break;
    case 2: q[0] = m02 - m20; q[1] = m10 + m01; q[2] = qa[2] * qa[2]; q[3] = m12 + m21; break;
    default: q[0] = m10 - m01; q[1] = m20 + m02; q[2] = m21 + m12; q[3] = qa[3] * qa[3]; break;
  }
  const float den = 2.0f * fmaxf(qa[best], 0.1f);
  const float sgn = (q[0] / den) < 0.f ? -1.f : 1.f;
  float* p = pose + (size_t)i * 9;
  for (int k = 0; k < 3; ++k) p[k] = T[(size_t)i * 3 + k];
  for (int k = 0; k < 4; ++k) p[3 + k] = sgn * (q[k] / den);
  for (int k = 0; k < 2; ++k) p[7 + k] = logf(fminf(fmaxf(F[(size_t)i * 2 + k], fmin), fmax)) - bias;
}
}  // namespace

extern "C" int pdb_camera_to_pose(pdb_context* c, const float* R_dev, const float* T_dev, const float* focal_dev, int32_t count,
                                  double log_focal_length_bias, double min_focal_length, double max_focal_length, float* pose_dev,
                                  void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (count < 0 || (count > 0 && (!R_dev || !T_dev || !focal_dev || !pose_dev))) return ctx->fail(PDB_ERR_INVALID, "bad argument");
  if (count == 0) return PDB_OK;
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  camera_to_pose_kernel<<<(count + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      R_dev, T_dev, focal_dev, count, (float)log_focal_length_bias, (float)min_focal_length, (float)max_focal_length, pose_dev);
  ctx->launches += 1;
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

extern "C" int pdb_dropout_mask_host(uint64_t seed, int32_t layer, int32_t site, int64_t offset, int64_t count, float dropout_p,
                                     uint8_t* out) {
  if (!out || count < 0 || offset < 0 || layer < 0 || layer >= kLayers || site < 0 || site > 3 || !(dropout_p >= 0.f && dropout_p < 1.f))
    return PDB_ERR_INVALID;
  const uint32_t th = dropout_threshold(dropout_p);
  for (int64_t i = 0; i < count; ++i) out[i] = dropout_keep(seed, layer, site, (uint64_t)(offset + i), th) ? 1 : 0;
  return PDB_OK;
}
