// Training entry points of the image backbone: the multi-scale DINO ViT-S/16 forward with explicit LayerNorm and every activation
// the backward needs saved in a caller-owned workspace, and the backward from dL/dz into the 150 parameter gradients.
//
// Same token layout as the inference path (csrc/api_vit.cu): the tokens of all scales and images form one [S, 384] matrix, so
// every projection, every dX = dY W and every dW = dY^T X is one wgmma/TMA GEMM (TF32 products, fp32 accumulate) without the
// split-K regime: each output element is one CTA's fixed-order dot product.  The 150 parameters are read where the caller holds
// them; nothing is folded or cached, so an optimizer step needs no reload.
//
// Saved per block: its input, (mean, rstd) of both norms, QKV, the attention output, the mid-block residual and the fc1
// pre-activation.  LayerNorm outputs, the GELU output and the attention probabilities are recomputed by the backward.
#include <vector>

#include "vit_train.cuh"

using namespace pdb;

namespace {

constexpr int kVitTrainMagic = 0x7d1a1e02;

struct VitTrainHeader {
  int32_t magic, n_images, height, width, n_scales, pad;
  double scales[kVitMaxScales];
};
static_assert(sizeof(VitTrainHeader) <= 64 * sizeof(float), "header fits the first 64 floats");

// Workspace: a 64-float header, the saved activations, then the backward's scratch.  Offsets in floats, each 64-float aligned.
struct VitTrainLayout {
  int n, S, Sp, n_scales;
  VitScale sc[kVitMaxScales];
  size_t cell[kVitMaxScales], weight[kVitMaxScales], pos[kVitMaxScales];
  size_t A, hin[kVitDepth + 1], st1[kVitDepth], qkv[kVitDepth], att[kVitDepth], hmid[kVitDepth], st2[kVitDepth], fc1[kVitDepth];
  size_t LNA, D0, D1, G1, PR, H, G2, T1, T2, Wt, part, HP, HB, PS[kVitMaxScales];
  size_t total;
  VitTrainLayout(int n_images, const VitScale* scales, int count, long long rows)
      : n(n_images), S((int)rows), Sp(((int)rows + 31) / 32 * 32), n_scales(count) {
    size_t at = 64;
    auto take = [&](size_t k) { size_t o = at; at += pad64(k); return o; };
    const size_t s = (size_t)S;
    for (int i = 0; i < count; ++i) {
      sc[i] = scales[i];
      cell[i] = take((size_t)kVitMaxTokens * kVitPosTaps);
      weight[i] = take((size_t)kVitMaxTokens * kVitPosTaps);
      pos[i] = take((size_t)sc[i].tokens * kVitDim);
    }
    A = take(s * kVitPatchK);
    for (int l = 0; l <= kVitDepth; ++l) hin[l] = take(s * kVitDim);
    for (int l = 0; l < kVitDepth; ++l) {
      st1[l] = take(2 * s); qkv[l] = take(s * 3 * kVitDim); att[l] = take(s * kVitDim); hmid[l] = take(s * kVitDim);
      st2[l] = take(2 * s); fc1[l] = take(s * kVitMlp);
    }
    LNA = take(s * kVitDim); D0 = take(s * kVitDim); D1 = take(s * kVitDim); G1 = take(s * kVitDim); PR = take(s * kVitDim);
    H = take(s * kVitMlp); G2 = take(s * kVitMlp);
    T1 = take((size_t)kVitMlp * Sp); T2 = take((size_t)kVitMlp * Sp); Wt = take((size_t)kVitMlp * kVitDim);
    part = take((size_t)kRedChunks * kVitMlp);
    HP = take((size_t)count * n * kVitDim); HB = take((size_t)count * n * kVitDim);
    for (int i = 0; i < count; ++i) PS[i] = take((size_t)sc[i].tokens * kVitDim);
    total = at;
  }
  // a scale reads the stored position table itself when dino's interpolate_pos_encoding would (196 patches of a square input)
  bool resampled(int i) const { return !(sc[i].gh == kVitGrid0 && sc[i].gw == kVitGrid0 && sc[i].out_h == sc[i].out_w); }
};

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_tensors(Context* ctx, const float* const* tensors, const char* what) {
  if (!tensors) return ctx->fail(PDB_ERR_INVALID, "%s is null", what);
  for (int i = 0; i < kVitTensors; ++i)
    if (!tensors[i] || !aligned16(tensors[i])) return ctx->fail(PDB_ERR_INVALID, "%s %d is null or not 16-byte aligned", what, i);
  return PDB_OK;
}

int gemm(Context* ctx, const float* X, const float* W, const float* bias, const float* residual, float* Y, int S, int O, int K,
         cudaStream_t st) {
  TcEpilogue E = {};
  E.bias = bias;
  E.residual = residual;
  E.ldr = O;
  E.Y = Y;
  E.ldy = O;
  E.S = S;
  E.O = O;
  E.K = K;
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

unsigned blocks(long long n, int per = 256) { return (unsigned)((n + per - 1) / per); }

}  // namespace

extern "C" int64_t pdb_vit_train_workspace_bytes(int32_t n_images, int32_t height, int32_t width, const double* scale_factors,
                                                 int32_t n_scales) {
  if (!scale_factors) return 0;
  VitScale sc[kVitMaxScales];
  long long rows = 0;
  char why[160];
  if (vit_plan_scales(n_images, height, width, scale_factors, n_scales, sc, &rows, why, sizeof(why)) != PDB_OK) return 0;
  return (int64_t)(VitTrainLayout(n_images, sc, n_scales, rows).total * sizeof(float));
}

extern "C" int pdb_vit_train_forward(pdb_context* c, const float* const* tensors, const float* images_dev, int32_t n_images,
                                     int32_t height, int32_t width, const double* scale_factors, int32_t n_scales, void* workspace,
                                     float* z_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (int rc = check_tensors(ctx, tensors, "parameter")) return rc;
  if (!images_dev || !z_dev || !scale_factors || !workspace) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (!aligned16(workspace) || !aligned16(images_dev)) return ctx->fail(PDB_ERR_INVALID, "workspace or images not 16-byte aligned");
  VitScale sc[kVitMaxScales];
  long long rows = 0;
  char why[160];
  if (int rc = vit_plan_scales(n_images, height, width, scale_factors, n_scales, sc, &rows, why, sizeof(why))) return ctx->fail(rc, "%s", why);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  VitTrainLayout L(n_images, sc, n_scales, rows);
  float* ws = static_cast<float*>(workspace);
  const int S = L.S;
  auto W = [&](int i) { return tensors[i]; };

  VitTrainHeader hdr = {};
  hdr.magic = kVitTrainMagic; hdr.n_images = n_images; hdr.height = height; hdr.width = width; hdr.n_scales = n_scales;
  for (int s = 0; s < n_scales; ++s) hdr.scales[s] = scale_factors[s];
  PDB_CUDA(ctx, cudaMemcpyAsync(ws, &hdr, sizeof(hdr), cudaMemcpyHostToDevice, st));
  // position tables: the stored one, or R_s applied to the caller's current pos_embed (the taps stay in the workspace for the adjoint)
  std::vector<int> cell;
  std::vector<float> weight;
  for (int s = 0; s < n_scales; ++s) {
    if (!L.resampled(s)) {
      L.sc[s].pos = W(1);
      continue;
    }
    const size_t taps = (size_t)(L.sc[s].tokens - 1) * kVitPosTaps;
    cell.resize(taps);
    weight.resize(taps);
    pos_taps(L.sc[s].gh, L.sc[s].gw, cell.data(), weight.data());
    PDB_CUDA(ctx, cudaMemcpyAsync(ws + L.cell[s], cell.data(), taps * sizeof(int), cudaMemcpyHostToDevice, st));
    PDB_CUDA(ctx, cudaMemcpyAsync(ws + L.weight[s], weight.data(), taps * sizeof(float), cudaMemcpyHostToDevice, st));
    PDB_CUDA(ctx, cudaStreamSynchronize(st));  // the host vectors are reused by the next scale
    vit_pos_apply_kernel<<<blocks((long long)L.sc[s].tokens * kVitDim), 256, 0, st>>>(
        W(1), reinterpret_cast<const int*>(ws + L.cell[s]), ws + L.weight[s], L.sc[s].tokens, ws + L.pos[s]);
    L.sc[s].pos = ws + L.pos[s];
    ctx->launches += 1;
  }
  // prepare_tokens
  for (int s = 0; s < n_scales; ++s)
    vit_patchify_kernel<<<dim3(L.sc[s].tokens, n_images), 256, 0, st>>>(images_dev, height, width, L.sc[s], ws + L.A);
  if (int rc = gemm(ctx, ws + L.A, W(2), W(3), nullptr, ws + L.hin[0], S, kVitDim, kVitPatchK, st)) return rc;
  for (int s = 0; s < n_scales; ++s) {
    const int total = n_images * L.sc[s].tokens * (kVitDim / 4);
    vit_pos_kernel<<<blocks(total), 256, 0, st>>>(ws + L.hin[0], L.sc[s], n_images, W(0));
  }
  const VitAttArgs att_args = vit_att_args(L.sc, n_scales, n_images);
  const long long nh = (long long)S * kVitMlp;
  for (int l = 0; l < kVitDepth; ++l) {
    const int b = 4 + 12 * l;  // norm1.{w,b} qkv.{w,b} proj.{w,b} norm2.{w,b} fc1.{w,b} fc2.{w,b}
    train_ln_fwd_kernel<kVitDim><<<blocks(S, 8), 256, 0, st>>>(ws + L.hin[l], W(b + 0), W(b + 1), S, kVitLnEps, ws + L.LNA, ws + L.st1[l]);
    if (int rc = gemm(ctx, ws + L.LNA, W(b + 2), W(b + 3), nullptr, ws + L.qkv[l], S, 3 * kVitDim, kVitDim, st)) return rc;
    if (int rc = enqueue_vit_attention(ctx, ws + L.qkv[l], ws + L.att[l], att_args, ctx->attr_vit_att[1], st)) return rc;
    if (int rc = gemm(ctx, ws + L.att[l], W(b + 4), W(b + 5), ws + L.hin[l], ws + L.hmid[l], S, kVitDim, kVitDim, st)) return rc;
    train_ln_fwd_kernel<kVitDim><<<blocks(S, 8), 256, 0, st>>>(ws + L.hmid[l], W(b + 6), W(b + 7), S, kVitLnEps, ws + L.LNA, ws + L.st2[l]);
    if (int rc = gemm(ctx, ws + L.LNA, W(b + 8), W(b + 9), nullptr, ws + L.fc1[l], S, kVitMlp, kVitDim, st)) return rc;
    vit_gelu_fwd_kernel<<<blocks(nh), 256, 0, st>>>(ws + L.fc1[l], ws + L.H, nh);
    if (int rc = gemm(ctx, ws + L.H, W(b + 10), W(b + 11), ws + L.hmid[l], ws + L.hin[l + 1], S, kVitDim, kVitMlp, st)) return rc;
  }
  vit_head_kernel<<<(n_images + 3) / 4, 128, 0, st>>>(ws + L.hin[kVitDepth], vit_head_args(L.sc, n_scales), W(4 + 12 * kVitDepth),
                                                      W(5 + 12 * kVitDepth), n_images, z_dev);
  ctx->launches += 2 * n_scales + kVitDepth * 4 + 1;
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

extern "C" int pdb_vit_backward(pdb_context* c, const float* const* tensors, void* workspace, const float* grad_z_dev,
                                float* const* grads, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (int rc = check_tensors(ctx, tensors, "parameter")) return rc;
  if (int rc = check_tensors(ctx, grads, "gradient")) return rc;
  if (!workspace || !grad_z_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  float* ws = static_cast<float*>(workspace);
  VitTrainHeader hdr;
  PDB_CUDA(ctx, cudaMemcpyAsync(&hdr, ws, sizeof(hdr), cudaMemcpyDeviceToHost, st));
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  VitScale sc[kVitMaxScales];
  long long rows = 0;
  char why[160];
  if (hdr.magic != kVitTrainMagic || hdr.n_scales < 1 || hdr.n_scales > kVitMaxScales ||
      vit_plan_scales(hdr.n_images, hdr.height, hdr.width, hdr.scales, hdr.n_scales, sc, &rows, why, sizeof(why)) != PDB_OK)
    return ctx->fail(PDB_ERR_STATE, "workspace does not hold a backbone training forward");
  const int n = hdr.n_images, n_scales = hdr.n_scales;
  const VitTrainLayout L(n, sc, n_scales, rows);
  const int S = L.S, Sp = L.Sp;
  auto W = [&](int i) { return tensors[i]; };
  auto G = [&](int i) { return grads[i]; };
  float *LNA = ws + L.LNA, *D0 = ws + L.D0, *D1 = ws + L.D1, *G1 = ws + L.G1, *PR = ws + L.PR, *H = ws + L.H, *G2 = ws + L.G2;
  float *T1 = ws + L.T1, *T2 = ws + L.T2, *Wt = ws + L.Wt, *part = ws + L.part;
  // dW[O, K] = dY[S, O]^T X[S, K] over the token-major transposes (zero-padded to Sp tokens)
  auto weight_grad = [&](const float* dY, int O, const float* X, int K, float* dW) {
    transpose(dY, S, O, Sp, T1, st);
    transpose(X, S, K, Sp, T2, st);
    return gemm(ctx, T1, T2, nullptr, nullptr, dW, O, K, Sp, st);
  };
  // dX[S, K] = dY[S, O] W[O, K] with W transposed to K-major
  auto input_grad = [&](const float* dY, const float* Wm, int O, int K, float* dX) {
    transpose(Wm, O, K, O, Wt, st);
    return gemm(ctx, dY, Wt, nullptr, nullptr, dX, S, K, O, st);
  };
  const size_t att_smem = vit_attn_bwd_smem(kVitMaxTokens);
  if (ctx->attr_vit_att[2] < att_smem) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(vit_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)att_smem));
    ctx->attr_vit_att[2] = att_smem;
  }
  // ---- head: only the class rows of the last residual stream receive gradient ----
  const int nb = 4 + 12 * kVitDepth;
  PDB_CUDA(ctx, cudaMemsetAsync(D0, 0, sizeof(float) * (size_t)S * kVitDim, st));
  vit_head_bwd_kernel<<<blocks((long long)n_scales * n, 4), 128, 0, st>>>(ws + L.hin[kVitDepth], vit_head_args(sc, n_scales), W(nb),
                                                                        grad_z_dev, n, D0, ws + L.HP, ws + L.HB);
  colsum(ws + L.HP, n_scales * n, kVitDim, part, G(nb), st);
  colsum(ws + L.HB, n_scales * n, kVitDim, part, G(nb + 1), st);
  const long long nh = (long long)S * kVitMlp;
  // ---- blocks, last first; D0 = gradient of the block output ----
  for (int l = kVitDepth - 1; l >= 0; --l) {
    const int b = 4 + 12 * l;
    vit_gelu_fwd_kernel<<<blocks(nh), 256, 0, st>>>(ws + L.fc1[l], H, nh);
    if (int rc = weight_grad(D0, kVitDim, H, kVitMlp, G(b + 10))) return rc;
    colsum(D0, S, kVitDim, part, G(b + 11), st);
    if (int rc = input_grad(D0, W(b + 10), kVitDim, kVitMlp, G2)) return rc;  // d gelu output
    vit_gelu_bwd_kernel<<<blocks(nh), 256, 0, st>>>(G2, ws + L.fc1[l], nh);   // d fc1 pre-activation
    train_ln_fwd_kernel<kVitDim><<<blocks(S, 8), 256, 0, st>>>(ws + L.hmid[l], W(b + 6), W(b + 7), S, kVitLnEps, LNA, ws + L.st2[l]);
    if (int rc = weight_grad(G2, kVitMlp, LNA, kVitDim, G(b + 8))) return rc;
    colsum(G2, S, kVitMlp, part, G(b + 9), st);
    if (int rc = input_grad(G2, W(b + 8), kVitMlp, kVitDim, G1)) return rc;  // d norm2 output
    train_ln_bwd_kernel<kVitDim><<<blocks(S, 8), 256, 0, st>>>(G1, ws + L.hmid[l], ws + L.st2[l], W(b + 6), D0, S, D1, PR);
    colsum(PR, S, kVitDim, part, G(b + 6), st);
    colsum(G1, S, kVitDim, part, G(b + 7), st);
    // D1 = gradient of the mid-block residual
    if (int rc = weight_grad(D1, kVitDim, ws + L.att[l], kVitDim, G(b + 4))) return rc;
    colsum(D1, S, kVitDim, part, G(b + 5), st);
    if (int rc = input_grad(D1, W(b + 4), kVitDim, kVitDim, G1)) return rc;  // d attention output
    float* dqkv = G2;
    for (int s = 0; s < n_scales; ++s)
      vit_attn_bwd_kernel<<<n * kVitHeads, 256, vit_attn_bwd_smem(sc[s].tokens), st>>>(ws + L.qkv[l], G1, sc[s].row0, sc[s].tokens, dqkv);
    train_ln_fwd_kernel<kVitDim><<<blocks(S, 8), 256, 0, st>>>(ws + L.hin[l], W(b + 0), W(b + 1), S, kVitLnEps, LNA, ws + L.st1[l]);
    if (int rc = weight_grad(dqkv, 3 * kVitDim, LNA, kVitDim, G(b + 2))) return rc;
    colsum(dqkv, S, 3 * kVitDim, part, G(b + 3), st);
    if (int rc = input_grad(dqkv, W(b + 2), 3 * kVitDim, kVitDim, G1)) return rc;  // d norm1 output
    train_ln_bwd_kernel<kVitDim><<<blocks(S, 8), 256, 0, st>>>(G1, ws + L.hin[l], ws + L.st1[l], W(b + 0), D1, S, D0, PR);
    colsum(PR, S, kVitDim, part, G(b + 0), st);
    colsum(G1, S, kVitDim, part, G(b + 1), st);
  }
  // ---- prepare_tokens: D0 = dX0.  Class rows of the im2col matrix are zero, so they add nothing to the patch weight gradient ----
  if (int rc = weight_grad(D0, kVitDim, ws + L.A, kVitPatchK, G(2))) return rc;
  VitPosGradArgs pa = {};
  pa.n_scales = n_scales;
  for (int s = 0; s < n_scales; ++s) {
    vit_pos_sum_kernel<<<blocks((long long)sc[s].tokens * kVitDim), 256, 0, st>>>(D0, sc[s].row0, sc[s].tokens, n, ws + L.PS[s]);
    pa.tokens[s] = sc[s].tokens;
    pa.resampled[s] = L.resampled(s);
    pa.sum[s] = ws + L.PS[s];
    pa.cell[s] = reinterpret_cast<const int*>(ws + L.cell[s]);
    pa.weight[s] = ws + L.weight[s];
  }
  vit_pos_grad_kernel<<<blocks((long long)(1 + kVitGrid0 * kVitGrid0) * kVitDim), 256, 0, st>>>(pa, G(1), G(0), G(3));
  ctx->launches += 6 + kVitDepth * (41 + n_scales) + 3 + n_scales + 1;
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}
