// Training entry points of the denoiser: GaussianDiffusion.p_losses forward with every activation the backward needs saved in a
// caller-owned workspace, the backward into 108 parameter gradients, the same pair for Denoiser.forward itself (eps from a given
// x, backward from dL/deps into the parameters, x and z), camera_to_pose_encoding, and the host image of the dropout masks.
// Projections run through enqueue_tc_linear (TF32 products, fp32 accumulate) without its split-K regime, so every output element
// is one CTA's fixed-order dot product; all other reductions are chunked fixed-order sums (csrc/train_common.cuh).
#include <cmath>
#include <cstring>

#include "denoiser.cuh"
#include "train.cuh"

using namespace pdb;

namespace {

constexpr int kMagic = 0x7d1a1e01;          // workspace filled by pdb_train_forward (p_losses)
constexpr int kMagicDenoiser = 0x7d1a1e02;  // workspace filled by pdb_denoiser_grad_forward (Denoiser.forward)

// Workspace: a 64-float header, the saved activations, then the backward's scratch.  Offsets in floats, each 64-float aligned.
struct TrainLayout {
  int B, N, S, Sp;
  size_t t, feed, u1, temb, hin[kLayers + 1], a1[kLayers], st1[kLayers], qkv[kLayers], P[kLayers], att[kLayers], hmid[kLayers],
      a2[kLayers], st2[kLayers], fd[kLayers], u, stu, r, diff;
  size_t D0, D1, G1, G2, T1, T2, Wt, part, Wpad, dWf, deps, dtemb, du1;
  size_t total;
  TrainLayout(int batch, int frames) : B(batch), N(frames), S(batch * frames), Sp((batch * frames + 31) / 32 * 32) {
    WorkspaceCursor cur;
    const size_t s = (size_t)S;
    t = cur.take(B);
    feed = cur.take(s * kFeedPad);
    u1 = cur.take((size_t)B * 128);
    temb = cur.take((size_t)B * 128);
    for (int l = 0; l <= kLayers; ++l) hin[l] = cur.take(s * kDM);
    for (int l = 0; l < kLayers; ++l) {
      a1[l] = cur.take(s * kDM); st1[l] = cur.take(2 * s); qkv[l] = cur.take(s * 3 * kDM); P[l] = cur.take((size_t)B * kHeads * N * N);
      att[l] = cur.take(s * kDM); hmid[l] = cur.take(s * kDM); a2[l] = cur.take(s * kDM); st2[l] = cur.take(2 * s); fd[l] = cur.take(s * kFF);
    }
    u = cur.take(s * kHid); stu = cur.take(2 * s); r = cur.take(s * kHid); diff = cur.take(s * 9);
    D0 = cur.take(s * kDM); D1 = cur.take(s * kDM); G1 = cur.take(s * 3 * kDM); G2 = cur.take(s * kFF);
    T1 = cur.take((size_t)3 * kDM * Sp); T2 = cur.take((size_t)kFF * Sp); Wt = cur.take((size_t)3 * kDM * kDM);
    part = cur.take((size_t)kRedChunks * 3 * kDM); Wpad = cur.take((size_t)kDM * kFeedPad); dWf = cur.take((size_t)kDM * kFeedPad);
    deps = cur.take(s * 9); dtemb = cur.take((size_t)B * 128); du1 = cur.take((size_t)B * 128);
    total = cur.at;
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

int check_params(Context* ctx, const float* const* params) {
  if (!params) return ctx->fail(PDB_ERR_INVALID, "params is null");
  for (int i = 0; i < PDB_NUM_WEIGHT_TENSORS; ++i) {
    if (!params[i]) return ctx->fail(PDB_ERR_INVALID, "parameter %d is null", i);
    if (!aligned16(params[i])) return ctx->fail(PDB_ERR_INVALID, "parameter %d is not 16-byte aligned", i);
  }
  return PDB_OK;
}

size_t attn_fwd_smem(int N) { return sizeof(float) * ((size_t)2 * N * 129 + 8 * 128 + 8 * 64); }
size_t attn_bwd_smem(int N) { return sizeof(float) * ((size_t)4 * N * 129 + (size_t)2 * N * (N + 1)); }

int set_attn_smem(Context* ctx) {
  if (!ctx->attr->train_att) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(train_attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_fwd_smem(kTrainMaxFrames)));
    PDB_CUDA(ctx, cudaFuncSetAttribute(train_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_bwd_smem(kTrainMaxFrames)));
    ctx->attr->train_att = true;
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

int check_forward_args(Context* ctx, int32_t batch, int32_t frames, float dropout_p, const void* workspace) {
  if (!aligned16(workspace)) return ctx->fail(PDB_ERR_INVALID, "workspace is not 16-byte aligned");
  if (batch < 1 || frames < 1) return ctx->fail(PDB_ERR_INVALID, "batch %d, frames %d", batch, frames);
  if (frames > kTrainMaxFrames) return ctx->fail(PDB_ERR_LIMIT, "training supports at most %d frames per sequence, got %d", kTrainMaxFrames, frames);
  if (!(dropout_p >= 0.f && dropout_p < 1.f)) return ctx->fail(PDB_ERR_INVALID, "dropout probability %g outside [0, 1)", (double)dropout_p);
  return PDB_OK;
}

// The forward both entry points share.  eps_mode (Denoiser.forward): the feed row is built from x_start = x, the tail writes eps
// into `loss`, and noise, x_t, x0 and the saved diff are not used; the header then carries kMagicDenoiser.
int enqueue_forward(Context* ctx, bool eps_mode, const float* const* params, const float* x_start, const int32_t* t, const float* noise,
                    const float* z, int32_t batch, int32_t frames, float dropout_p, uint64_t seed, int32_t loss_type, void* workspace,
                    float* loss, float* x_t, float* x0, cudaStream_t st) {
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (int rc = set_attn_smem(ctx)) return rc;
  const TrainLayout L(batch, frames);
  float* ws = static_cast<float*>(workspace);
  const int S = L.S, B = batch, N = frames;
  const TrainSched sc = train_schedule();
  const DropCfg d = drop_cfg(dropout_threshold(dropout_p), 1.0f / (1.0f - dropout_p), seed);
  int* tsv = reinterpret_cast<int*>(ws + L.t);
  TrainHeader hdr = {eps_mode ? kMagicDenoiser : kMagic, batch, frames, loss_type, d.threshold, (uint32_t)seed, (uint32_t)(seed >> 32),
                     d.scale, 0};
  train_launch(ctx, st, train_header_kernel, 1, 128, 0, hdr, reinterpret_cast<int*>(ws), t, tsv);
  auto W = [&](int i) { return params[i]; };
  // feed
  train_launch(ctx, st, train_time_mlp_kernel, B, 128, 0, tsv, W(0), W(1), W(2), W(3), ws + L.u1, ws + L.temb);
  if (eps_mode)
    train_launch(ctx, st, train_feed_kernel<true>, S, 256, 0, sc, x_start, nullptr, tsv, ws + L.temb, z, N, S, nullptr, ws + L.feed);
  else
    train_launch(ctx, st, train_feed_kernel<false>, S, 256, 0, sc, x_start, noise, tsv, ws + L.temb, z, N, S, x_t, ws + L.feed);
  train_launch(ctx, st, train_copy_cols_kernel, blocks((long long)kDM * kFeedPad), 256, 0, W(4), kFirstIn, kDM, kFirstIn, ws + L.Wpad,
               kFeedPad);
  if (int rc = train_gemm(ctx, ws + L.feed, ws + L.Wpad, W(5), nullptr, ws + L.hin[0], S, kDM, kFeedPad, 0, st)) return rc;
  const long long nd = (long long)S * kDM, nf = (long long)S * kFF;
  for (int l = 0; l < kLayers; ++l) {
    const int b = 6 + 12 * l;
    train_launch(ctx, st, train_ln_fwd_kernel<kDM>, blocks(S, 8), 256, 0, ws + L.hin[l], W(b + 8), W(b + 9), S, kLnEps, ws + L.a1[l],
                 ws + L.st1[l]);
    if (int rc = train_gemm(ctx, ws + L.a1[l], W(b + 0), W(b + 1), nullptr, ws + L.qkv[l], S, 3 * kDM, kDM, 0, st)) return rc;
    train_launch(ctx, st, train_attn_fwd_kernel, B * kHeads, 256, attn_fwd_smem(N), ws + L.qkv[l], N, d, l, ws + L.P[l], ws + L.att[l]);
    if (int rc = train_gemm(ctx, ws + L.att[l], W(b + 2), W(b + 3), nullptr, ws + L.G1, S, kDM, kDM, 0, st)) return rc;
    train_launch(ctx, st, train_dropout_kernel, blocks(nd), 256, 0, ws + L.G1, ws + L.hin[l], nullptr, ws + L.hmid[l], nd, d, l, kSiteOut);
    train_launch(ctx, st, train_ln_fwd_kernel<kDM>, blocks(S, 8), 256, 0, ws + L.hmid[l], W(b + 10), W(b + 11), S, kLnEps, ws + L.a2[l],
                 ws + L.st2[l]);
    if (int rc = train_gemm(ctx, ws + L.a2[l], W(b + 4), W(b + 5), nullptr, ws + L.fd[l], S, kFF, kDM, 1, st)) return rc;
    train_launch(ctx, st, train_dropout_kernel, blocks(nf), 256, 0, ws + L.fd[l], nullptr, nullptr, ws + L.fd[l], nf, d, l, kSiteRelu);
    if (int rc = train_gemm(ctx, ws + L.fd[l], W(b + 6), W(b + 7), nullptr, ws + L.G1, S, kDM, kFF, 0, st)) return rc;
    train_launch(ctx, st, train_dropout_kernel, blocks(nd), 256, 0, ws + L.G1, ws + L.hmid[l], nullptr, ws + L.hin[l + 1], nd, d, l,
                 kSiteFF2);
  }
  const int tb = 6 + 12 * kLayers;
  if (int rc = train_gemm(ctx, ws + L.hin[kLayers], W(tb), W(tb + 1), nullptr, ws + L.u, S, kHid, kDM, 0, st)) return rc;
  if (eps_mode)
    train_launch(ctx, st, train_tail_fwd_kernel<true>, blocks(S, 8), 256, 0, sc, ws + L.u, W(tb + 2), W(tb + 3), W(tb + 4), W(tb + 5), tsv,
                 nullptr, nullptr, N, S, 0, ws + L.stu, ws + L.r, nullptr, loss, nullptr);
  else
    train_launch(ctx, st, train_tail_fwd_kernel<false>, blocks(S, 8), 256, 0, sc, ws + L.u, W(tb + 2), W(tb + 3), W(tb + 4), W(tb + 5), tsv,
                 x_t, noise, N, S, loss_type, ws + L.stu, ws + L.r, ws + L.diff, loss, x0);
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

// The backward both entry points share, from the workspace a forward with header magic `magic` filled.  grad_loss / grad_x0 seed the
// tail as in p_losses; with magic == kMagicDenoiser grad_loss is dL/deps.  grads == NULL runs only the input-gradient chain (dropout,
// linear-layer input gradients, LayerNorm and attention backward) towards grad_x / grad_z; each of those may be NULL.
int enqueue_backward(Context* ctx, int magic, const float* const* params, void* workspace, const float* grad_loss, const float* grad_x0,
                     float* const* grads, float* grad_x, float* grad_z, cudaStream_t st) {
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (int rc = set_attn_smem(ctx)) return rc;
  float* ws = static_cast<float*>(workspace);
  TrainHeader hdr;
  PDB_CUDA(ctx, cudaMemcpyAsync(&hdr, ws, sizeof(hdr), cudaMemcpyDeviceToHost, st));
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  if (hdr.magic != magic || hdr.batch < 1 || hdr.frames < 1 || hdr.frames > kTrainMaxFrames)
    return ctx->fail(PDB_ERR_STATE, magic == kMagic ? "workspace does not hold a training forward"
                                                    : "workspace does not hold a pdb_denoiser_grad_forward");
  if (hdr.bad_t) return ctx->fail(PDB_ERR_INVALID, "the forward was given a timestep outside [0, %d)", kT);
  const bool eps_mode = magic == kMagicDenoiser;
  const TrainLayout L(hdr.batch, hdr.frames);
  const int S = L.S, B = hdr.batch, N = hdr.frames;
  const TrainSched sc = train_schedule();
  const DropCfg d = drop_cfg(hdr.threshold, hdr.scale, (uint64_t)hdr.seed_lo | ((uint64_t)hdr.seed_hi << 32));
  const int* tsv = reinterpret_cast<const int*>(ws + L.t);
  auto W = [&](int i) { return params[i]; };
  auto G = [&](int i) { return grads[i]; };
  float *D0 = ws + L.D0, *D1 = ws + L.D1, *G1 = ws + L.G1, *G2 = ws + L.G2, *part = ws + L.part;
  const LinearGrad lin = {ctx, S, L.Sp, ws + L.T1, ws + L.T2, ws + L.Wt, part, st};
  const long long nd = (long long)S * kDM, nf = (long long)S * kFF;
  // ---- tail ----
  const int tb = 6 + 12 * kLayers;
  float* dau = G2;  // [S, 128]
  if (eps_mode)
    train_launch(ctx, st, train_tail_bwd_kernel<true>, blocks(S, 8), 256, 0, sc, nullptr, grad_loss, nullptr, tsv, N, S, 0, W(tb + 4),
                 ws + L.r, ws + L.deps, dau);
  else
    train_launch(ctx, st, train_tail_bwd_kernel<false>, blocks(S, 8), 256, 0, sc, ws + L.diff, grad_loss, grad_x0, tsv, N, S,
                 hdr.loss_type, W(tb + 4), ws + L.r, ws + L.deps, dau);
  if (grads) {
    train_launch(ctx, st, train_w3_partial_kernel, kRedChunks, 128, 0, ws + L.deps, ws + L.r, S, part);
    train_launch(ctx, st, train_chunk_sum_kernel, blocks(9 * 128), 256, 0, part, kRedChunks, 9 * 128, G(tb + 4));
    lin.bias(ws + L.deps, S, 9, G(tb + 5));
  }
  float* du = G1;  // [S, 128]
  train_launch(ctx, st, train_ln_bwd_kernel<kHid>, blocks(S, 8), 256, 0, dau, ws + L.u, ws + L.stu, W(tb + 2), nullptr, S, du,
               G2 + (size_t)S * kHid);
  if (grads) {
    lin.bias(G2 + (size_t)S * kHid, S, kHid, G(tb + 2));
    lin.bias(dau, S, kHid, G(tb + 3));
    if (int rc = lin.weight(du, kHid, ws + L.hin[kLayers], kDM, G(tb))) return rc;
    lin.bias(du, S, kHid, G(tb + 1));
  }
  if (int rc = lin.input(du, W(tb), kHid, kDM, D0)) return rc;
  // ---- trunk, last layer first; D0 = gradient of the layer output ----
  for (int l = kLayers - 1; l >= 0; --l) {
    const int b = 6 + 12 * l;
    float* dy2 = G1;
    train_launch(ctx, st, train_dropout_kernel, blocks(nd), 256, 0, D0, nullptr, nullptr, dy2, nd, d, l, kSiteFF2);
    if (int rc = lin.input(dy2, W(b + 6), kDM, kFF, G2)) return rc;  // d fd
    if (grads) {
      if (int rc = lin.weight(dy2, kDM, ws + L.fd[l], kFF, G(b + 6))) return rc;
      lin.bias(dy2, S, kDM, G(b + 7));
    }
    train_launch(ctx, st, train_dropout_kernel, blocks(nf), 256, 0, G2, nullptr, ws + L.fd[l], G2, nf, d, l, kSiteRelu);  // d(FF1 output)
    float* da2 = G1;
    if (int rc = lin.input(G2, W(b + 4), kFF, kDM, da2)) return rc;
    if (grads) {
      if (int rc = lin.weight(G2, kFF, ws + L.a2[l], kDM, G(b + 4))) return rc;
      lin.bias(G2, S, kFF, G(b + 5));
    }
    train_launch(ctx, st, train_ln_bwd_kernel<kDM>, blocks(S, 8), 256, 0, da2, ws + L.hmid[l], ws + L.st2[l], W(b + 10), D0, S, D1, G2);
    if (grads) {
      lin.bias(G2, S, kDM, G(b + 10));
      lin.bias(da2, S, kDM, G(b + 11));
    }
    float* dy = G1;
    train_launch(ctx, st, train_dropout_kernel, blocks(nd), 256, 0, D1, nullptr, nullptr, dy, nd, d, l, kSiteOut);
    if (int rc = lin.input(dy, W(b + 2), kDM, kDM, G2)) return rc;  // d att
    if (grads) {
      if (int rc = lin.weight(dy, kDM, ws + L.att[l], kDM, G(b + 2))) return rc;
      lin.bias(dy, S, kDM, G(b + 3));
    }
    float* dqkv = G1;
    train_launch(ctx, st, train_attn_bwd_kernel, B * kHeads, 256, attn_bwd_smem(N), ws + L.qkv[l], ws + L.P[l], G2, N, d, l, dqkv);
    float* da1 = G2;
    if (int rc = lin.input(dqkv, W(b + 0), 3 * kDM, kDM, da1)) return rc;
    if (grads) {
      if (int rc = lin.weight(dqkv, 3 * kDM, ws + L.a1[l], kDM, G(b + 0))) return rc;
      lin.bias(dqkv, S, 3 * kDM, G(b + 1));
    }
    train_launch(ctx, st, train_ln_bwd_kernel<kDM>, blocks(S, 8), 256, 0, da1, ws + L.hin[l], ws + L.st1[l], W(b + 8), D1, S, D0, G1);
    if (grads) {
      lin.bias(G1, S, kDM, G(b + 8));
      lin.bias(da1, S, kDM, G(b + 9));
    }
  }
  // ---- _first and the time MLP ----
  if (grads) {
    if (int rc = lin.weight(D0, kDM, ws + L.feed, kFeedPad, ws + L.dWf)) return rc;
    train_launch(ctx, st, train_copy_cols_kernel, blocks((long long)kDM * kFirstIn), 256, 0, ws + L.dWf, kFeedPad, kDM, kFirstIn, G(4),
                 kFirstIn);
    lin.bias(D0, S, kDM, G(5));
    train_launch(ctx, st, train_dtemb_kernel, B, 256, 0, D0, N, W(4), ws + L.dtemb);
    train_launch(ctx, st, train_time_du_kernel, blocks((long long)B * 128), 256, 0, ws + L.dtemb, ws + L.u1, W(2), B, ws + L.du1);
    train_launch(ctx, st, train_time_dw_kernel, blocks(128 * 128), 256, 0, ws + L.dtemb, ws + L.u1, tsv, B, 128, 1, G(2), G(3));
    train_launch(ctx, st, train_time_dw_kernel, blocks(128 * 256), 256, 0, ws + L.du1, ws + L.u1, tsv, B, 256, 0, G(0), G(1));
  }
  if (grad_z) {
    // dz = dh0 . W_first[:, 317:701]: the column block starts at float 317, which TMA cannot address, so it is copied to an
    // aligned [512, 384] buffer (the _first weight-gradient staging area, free by now) and then read K-major like every dX
    float* Wz = ws + L.dWf;
    train_launch(ctx, st, train_copy_cols_kernel, blocks((long long)kDM * kZ), 256, 0, W(4) + 317, kFirstIn, kDM, kZ, Wz, kZ);
    if (int rc = lin.input(D0, Wz, kDM, kZ, grad_z)) return rc;
  }
  if (grad_x) {
    // dfeed[:, 0:189] = dh0 . W_first[:, 0:189] through the same staging area (zero-padded to 192 columns, the GEMM's 64-multiple),
    // into G1 (free after the trunk); then the harmonic embedding's chain rule per element
    constexpr int kXCols = 189, kXPad = 192;
    float* Wx = ws + L.dWf;
    train_launch(ctx, st, train_copy_cols_kernel, blocks((long long)kDM * kXPad), 256, 0, W(4), kFirstIn, kDM, kXCols, Wx, kXPad);
    if (int rc = lin.input(D0, Wx, kDM, kXPad, G1)) return rc;
    train_launch(ctx, st, train_dx_kernel, blocks((long long)S * 9), 256, 0, ws + L.feed, G1, S, grad_x);
  }
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

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
  if (int rc = check_forward_args(ctx, batch, frames, dropout_p, workspace)) return rc;
  if (loss_type != 0 && loss_type != 1) return ctx->fail(PDB_ERR_INVALID, "loss_type %d (0 = l1, 1 = l2)", loss_type);
  return enqueue_forward(ctx, false, params, x_start, t, noise, z, batch, frames, dropout_p, seed, loss_type, workspace, loss, x_t, x0,
                         static_cast<cudaStream_t>(stream));
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
  return enqueue_backward(ctx, kMagic, params, workspace, grad_loss, grad_x0, grads, nullptr, grad_z, static_cast<cudaStream_t>(stream));
}

extern "C" int pdb_denoiser_grad_forward(pdb_context* c, const float* const* params, const float* x, const int32_t* t, const float* z,
                                         int32_t batch, int32_t frames, float dropout_p, uint64_t seed, void* workspace, float* eps,
                                         void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (int rc = check_params(ctx, params)) return rc;
  if (!x || !t || !z || !workspace || !eps) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (int rc = check_forward_args(ctx, batch, frames, dropout_p, workspace)) return rc;
  return enqueue_forward(ctx, true, params, x, t, nullptr, z, batch, frames, dropout_p, seed, 0, workspace, eps, nullptr, nullptr,
                         static_cast<cudaStream_t>(stream));
}

extern "C" int pdb_denoiser_grad_backward(pdb_context* c, const float* const* params, void* workspace, const float* grad_eps,
                                          float* const* grads, float* grad_x, float* grad_z, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (int rc = check_params(ctx, params)) return rc;
  if (!workspace || !grad_eps) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (!grads && !grad_x && !grad_z) return ctx->fail(PDB_ERR_INVALID, "no gradient requested");
  if ((grad_x && !aligned16(grad_x)) || (grad_z && !aligned16(grad_z)))
    return ctx->fail(PDB_ERR_INVALID, "grad_x or grad_z is not 16-byte aligned");
  if (grads)
    for (int i = 0; i < PDB_NUM_WEIGHT_TENSORS; ++i)
      if (!grads[i] || !aligned16(grads[i])) return ctx->fail(PDB_ERR_INVALID, "gradient %d is null or not 16-byte aligned", i);
  return enqueue_backward(ctx, kMagicDenoiser, params, workspace, grad_eps, nullptr, grads, grad_x, grad_z,
                          static_cast<cudaStream_t>(stream));
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
  train_launch(ctx, static_cast<cudaStream_t>(stream), camera_to_pose_kernel, (count + 127) / 128, 128, 0, R_dev, T_dev, focal_dev, count,
               (float)log_focal_length_bias, (float)min_focal_length, (float)max_focal_length, pose_dev);
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
