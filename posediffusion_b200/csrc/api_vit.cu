// Image features z = MultiScaleImageFeatureExtractor(image) (reference: models/image_feature_extractor.py:27-87): DINO ViT-S/16
// (torch.hub facebookresearch/dino:main `vit_small(patch_size=16)`, restated in oracle/dino_vit.py) applied to the ResNet-normalised
// image at every scale factor, class-token features averaged over the scales.
//
// Layout: the tokens of ALL scales and images form one [S_total, 384] activation matrix (scale-major, then image, then
// token; 197 + 50 + 17 tokens per 224^2 image at the default scales), so that every projection of a block is ONE wgmma/TMA
// GEMM (csrc/tc_linear.cuh, TF32 products, fp32 accumulate) over all of them:
//   patchify (normalise + bilinear resize + im2col, fused) -> GEMM [S,768]x[768,384] -> + class token / position table
//   12 x { row stats -> GEMM qkv (LayerNorm folded into the weights, applied in the epilogue) -> attention (shared memory,
//          4 query rows per warp) -> GEMM proj (+residual) -> row stats -> GEMM fc1 (folded LN, exact GELU) -> GEMM fc2 (+residual) }
//   head: final LayerNorm of the class rows, summed over scales in the reference's order, divided by the number of scales.
#include <new>

#include "fold_ln.cuh"
#include "vit.cuh"

using namespace pdb;

namespace pdb {
void vit_release(Context* ctx) {
  if (!ctx->vit) return;
  for (auto& e : ctx->vit->pos_tables) cudaFree(std::get<2>(e));
  if (ctx->vit->arena) cudaFree(ctx->vit->arena);
  delete ctx->vit;
  ctx->vit = nullptr;
  if (ctx->vit_ws) cudaFree(ctx->vit_ws);
  ctx->vit_ws = nullptr;
  ctx->vit_ws_bytes = 0;
}
}  // namespace pdb

extern "C" int pdb_vit_pos_table(const float* pos_embed_host, int32_t grid_h, int32_t grid_w, float* out_host) {
  if (!pos_embed_host || !out_host || grid_h < 1 || grid_w < 1) return PDB_ERR_INVALID;
  if (grid_h == kVitGrid0 && grid_w == kVitGrid0) {
    std::memcpy(out_host, pos_embed_host, sizeof(float) * (1 + kVitGrid0 * kVitGrid0) * kVitDim);
    return PDB_OK;
  }
  resample_pos(pos_embed_host, grid_h, grid_w, out_host);
  return PDB_OK;
}

extern "C" int pdb_vit_load(pdb_context* c, const float* const* tensors, const int64_t* numels, int32_t count, int32_t on_device,
                            void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!tensors || !numels) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (count != kVitTensors) return ctx->fail(PDB_ERR_INVALID, "expected %d tensors of dino_vits16, got %d", kVitTensors, count);
  for (int i = 0; i < count; ++i)
    if (!tensors[i] || numels[i] != (int64_t)vit_tensor_floats(i))
      return ctx->fail(PDB_ERR_INVALID, "tensor %d: expected %lld elements, got %lld", i, (long long)vit_tensor_floats(i), (long long)numels[i]);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  vit_release(ctx);
  VitWeights* w = new (std::nothrow) VitWeights();
  if (!w) return ctx->fail(PDB_ERR_CUDA, "out of host memory");
  std::vector<size_t> off(count);
  size_t total = 0;
  for (int i = 0; i < count; ++i) {
    off[i] = total;
    total += pad64(vit_tensor_floats(i));
  }
  // folded copies: per layer qkv weight + bias + colsum, fc1 weight + bias + colsum
  const size_t fold_layer = pad64((size_t)3 * kVitDim * kVitDim) + 2 * pad64(3 * kVitDim) + pad64((size_t)kVitMlp * kVitDim) + 2 * pad64(kVitMlp);
  const size_t fold0 = total;
  total += fold_layer * kVitDepth;
  cudaError_t err = cudaMalloc(&w->arena, total * sizeof(float));
  if (err != cudaSuccess) {
    delete w;
    return ctx->fail(PDB_ERR_CUDA, "cudaMalloc(%zu) failed: %s", total * sizeof(float), cudaGetErrorString(err));
  }
  ctx->vit = w;
  float* A = w->arena;
  for (int i = 0; i < count; ++i)
    PDB_CUDA(ctx, cudaMemcpyAsync(A + off[i], tensors[i], vit_tensor_floats(i) * sizeof(float),
                                  on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  w->pos_host.resize(vit_tensor_floats(1));
  PDB_CUDA(ctx, cudaMemcpyAsync(w->pos_host.data(), A + off[1], vit_tensor_floats(1) * sizeof(float), cudaMemcpyDeviceToHost, st));
  w->cls = A + off[0];
  w->pos = A + off[1];
  w->wpatch = A + off[2];
  w->bpatch = A + off[3];
  w->norm_g = A + off[4 + 12 * kVitDepth];
  w->norm_b = A + off[5 + 12 * kVitDepth];
  for (int l = 0; l < kVitDepth; ++l) {
    const int b = 4 + 12 * l;  // norm1.{w,b} qkv.{w,b} proj.{w,b} norm2.{w,b} fc1.{w,b} fc2.{w,b}
    float* f = A + fold0 + fold_layer * l;
    float* wqkv = f;          f += pad64((size_t)3 * kVitDim * kVitDim);
    float* bias_qkv = f;      f += pad64(3 * kVitDim);
    float* colsum_qkv = f;    f += pad64(3 * kVitDim);
    float* wfc1 = f;          f += pad64((size_t)kVitMlp * kVitDim);
    float* bias_fc1 = f;      f += pad64(kVitMlp);
    float* colsum_fc1 = f;
    fold_ln_kernel<<<3 * kVitDim, 128, 0, st>>>(A + off[b + 2], A + off[b + 3], A + off[b + 0], A + off[b + 1], kVitDim, wqkv, colsum_qkv, bias_qkv);
    fold_ln_kernel<<<kVitMlp, 128, 0, st>>>(A + off[b + 8], A + off[b + 9], A + off[b + 6], A + off[b + 7], kVitDim, wfc1, colsum_fc1, bias_fc1);
    VitLayer& L = w->layer[l];
    L.wqkv = wqkv; L.bias_qkv = bias_qkv; L.colsum_qkv = colsum_qkv;
    L.wproj = A + off[b + 4]; L.bproj = A + off[b + 5];
    L.wfc1 = wfc1; L.bias_fc1 = bias_fc1; L.colsum_fc1 = colsum_fc1;
    L.wfc2 = A + off[b + 10]; L.bfc2 = A + off[b + 11];
  }
  PDB_CUDA(ctx, cudaGetLastError());
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  ctx->launches += 2 * kVitDepth;
  return PDB_OK;
}

extern "C" int pdb_extract_features(pdb_context* c, const float* images_dev, int32_t n_images, int32_t height, int32_t width,
                                    const double* scale_factors, int32_t n_scales, float* z_dev, float* tokens_debug_dev,
                                    int32_t debug_stage, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!images_dev || !z_dev || !scale_factors) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (!ctx->vit) return ctx->fail(PDB_ERR_STATE, "image backbone weights not loaded (pdb_vit_load)");
  VitScale sc[kVitMaxScales];
  long long rows = 0;
  char why[160];
  if (int rc = vit_plan_scales(n_images, height, width, scale_factors, n_scales, sc, &rows, why, sizeof(why))) return ctx->fail(rc, "%s", why);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  VitWeights* w = ctx->vit;
  for (int s = 0; s < n_scales; ++s)
    if (int rc = vit_pos_table(ctx, w, sc[s].gh, sc[s].gw, sc[s].out_h == sc[s].out_w, &sc[s].pos, st)) return rc;
  const VitHeadArgs head = vit_head_args(sc, n_scales);
  const int S = (int)rows;
  // workspace: X [S,384] | QKV [S,1152] | ATT [S,384] | HID [S,1536] (the im2col matrix [S,768] aliases HID) | mean, rstd [S]
  const size_t need = sizeof(float) * ((size_t)S * (kVitDim + 3 * kVitDim + kVitDim + kVitMlp) + 2 * pad64(S) + 64);
  if (int rc = ensure_buffer(ctx, &ctx->vit_ws, &ctx->vit_ws_bytes, need)) return rc;
  float* X = static_cast<float*>(ctx->vit_ws);
  float* QKV = X + (size_t)S * kVitDim;
  float* ATT = QKV + (size_t)S * 3 * kVitDim;
  float* HID = ATT + (size_t)S * kVitDim;
  float* mean = HID + (size_t)S * kVitMlp;
  float* rstd = mean + pad64(S);
  float* Apatch = HID;

  const VitAttArgs att_args = vit_att_args(sc, n_scales, n_images);
  auto lin = [&](const float* in, const float* Wm, int O, int K, const float* bias, const float* residual, const float* colsum, float* Y,
                 int gelu) {
    TcEpilogue E = {};
    E.bias = bias; E.residual = residual; E.ldr = O;
    E.colsum = colsum; E.row_mean = colsum ? mean : nullptr; E.row_rstd = colsum ? rstd : nullptr;
    E.Y = Y; E.ldy = O; E.S = S; E.O = O; E.K = K; E.gelu = gelu;
    return enqueue_tc_linear(ctx, in, Wm, E, st);
  };
  auto dump = [&](int stage) -> int {
    if (tokens_debug_dev && debug_stage == stage)
      PDB_CUDA(ctx, cudaMemcpyAsync(tokens_debug_dev, X, sizeof(float) * (size_t)S * kVitDim, cudaMemcpyDeviceToDevice, st));
    return PDB_OK;
  };
  int rc = PDB_OK;
  for (int s = 0; s < n_scales; ++s) {
    vit_patchify_kernel<<<dim3(sc[s].tokens, n_images), 256, 0, st>>>(images_dev, height, width, sc[s], Apatch);
    ctx->launches += 1;
  }
  rc = lin(Apatch, w->wpatch, kVitDim, kVitPatchK, w->bpatch, nullptr, nullptr, X, 0);
  for (int s = 0; s < n_scales && rc == PDB_OK; ++s) {
    const int total = n_images * sc[s].tokens * (kVitDim / 4);
    vit_pos_kernel<<<(total + 255) / 256, 256, 0, st>>>(X, sc[s], n_images, w->cls);
    ctx->launches += 1;
  }
  if (rc == PDB_OK) rc = dump(0);
  for (int l = 0; l < kVitDepth && rc == PDB_OK; ++l) {
    const VitLayer& L = w->layer[l];
    vit_row_stats_kernel<<<(S + 7) / 8, 256, 0, st>>>(X, mean, rstd, S);
    if ((rc = lin(X, L.wqkv, 3 * kVitDim, kVitDim, L.bias_qkv, nullptr, L.colsum_qkv, QKV, 0))) break;
    if ((rc = enqueue_vit_attention(ctx, QKV, ATT, att_args, ctx->attr->vit_att[0], st))) break;
    if ((rc = lin(ATT, L.wproj, kVitDim, kVitDim, L.bproj, X, nullptr, X, 0))) break;
    vit_row_stats_kernel<<<(S + 7) / 8, 256, 0, st>>>(X, mean, rstd, S);
    if ((rc = lin(X, L.wfc1, kVitMlp, kVitDim, L.bias_fc1, nullptr, L.colsum_fc1, HID, 1))) break;
    if ((rc = lin(HID, L.wfc2, kVitDim, kVitMlp, L.bfc2, X, nullptr, X, 0))) break;
    ctx->launches += 3;
    rc = dump(l + 1);
  }
  if (rc != PDB_OK) return rc;
  vit_head_kernel<<<(n_images + 3) / 4, 128, 0, st>>>(X, head, w->norm_g, w->norm_b, n_images, z_dev);
  ctx->launches += 1;
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

extern "C" int pdb_extract_features_host(pdb_context* c, const float* images_host, int32_t n_images, int32_t height, int32_t width,
                                         const double* scale_factors, int32_t n_scales, float* z_host, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!images_host || !z_host) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (n_images < 1 || height < 1 || width < 1) return ctx->fail(PDB_ERR_INVALID, "bad image batch [%d,3,%d,%d]", n_images, height, width);
  if (n_images > kVitMaxImages) return ctx->fail(PDB_ERR_LIMIT, "%d images in one call (limit %d)", n_images, kVitMaxImages);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t img_bytes = sizeof(float) * (size_t)n_images * 3 * height * width, z_bytes = sizeof(float) * (size_t)n_images * kVitDim;
  if (int rc = ensure_buffer(ctx, &ctx->stage, &ctx->stage_bytes, img_bytes + z_bytes + 256)) return rc;
  float* img_dev = static_cast<float*>(ctx->stage);
  float* z_dev = reinterpret_cast<float*>(static_cast<char*>(ctx->stage) + ((img_bytes + 255) & ~(size_t)255));
  PDB_CUDA(ctx, cudaMemcpyAsync(img_dev, images_host, img_bytes, cudaMemcpyHostToDevice, st));
  if (int rc = pdb_extract_features(c, img_dev, n_images, height, width, scale_factors, n_scales, z_dev, nullptr, 0, stream)) return rc;
  PDB_CUDA(ctx, cudaMemcpyAsync(z_host, z_dev, z_bytes, cudaMemcpyDeviceToHost, st));
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  return PDB_OK;
}
