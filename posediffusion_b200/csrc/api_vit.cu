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
#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <tuple>
#include <vector>

#include "context.cuh"
#include "fold_ln.cuh"
#include "tc_linear.cuh"

using namespace pdb;

namespace pdb {

constexpr int kVitDim = 384, kVitHeads = 6, kVitHD = 64, kVitDepth = 12, kVitMlp = 1536, kVitPatch = 16;
constexpr int kVitPatchK = 3 * kVitPatch * kVitPatch;  // 768
constexpr int kVitGrid0 = 14;                          // native 224 / 16 position grid
constexpr int kVitMaxTokens = 256;                     // tokens per (image, scale) the attention kernel keeps in shared memory
constexpr int kVitMaxScales = 4;
constexpr float kVitLnEps = 1e-6f;
constexpr int kVitTensors = 4 + 12 * kVitDepth + 2;

struct VitLayer {
  const float *wqkv, *bias_qkv, *colsum_qkv;  // norm1 folded in
  const float *wproj, *bproj;
  const float *wfc1, *bias_fc1, *colsum_fc1;  // norm2 folded in
  const float *wfc2, *bfc2;
};
struct VitWeights {
  float* arena = nullptr;
  const float *cls = nullptr, *pos = nullptr, *wpatch = nullptr, *bpatch = nullptr, *norm_g = nullptr, *norm_b = nullptr;
  VitLayer layer[kVitDepth];
  std::vector<float> pos_host;                             // [197, 384] for resampling on the host
  std::vector<std::tuple<int, int, float*>> pos_tables;    // (grid_h, grid_w) -> device [1 + gh*gw, 384]
};

}  // namespace pdb

namespace {

size_t vit_tensor_floats(int i) {
  if (i == 0) return kVitDim;
  if (i == 1) return (size_t)(1 + kVitGrid0 * kVitGrid0) * kVitDim;
  if (i == 2) return (size_t)kVitDim * kVitPatchK;
  if (i == 3) return kVitDim;
  if (i >= 4 + 12 * kVitDepth) return kVitDim;
  switch ((i - 4) % 12) {
    case 0: case 1: case 6: case 7: return kVitDim;  // norm1 / norm2
    case 2: return (size_t)3 * kVitDim * kVitDim;
    case 3: return 3 * kVitDim;
    case 4: return (size_t)kVitDim * kVitDim;
    case 5: return kVitDim;
    case 8: return (size_t)kVitMlp * kVitDim;
    case 9: return kVitMlp;
    case 10: return (size_t)kVitDim * kVitMlp;
    default: return kVitDim;
  }
}
inline size_t pad64(size_t n) { return (n + 63) & ~(size_t)63; }

// ---- torch.nn.functional.interpolate(mode="bicubic", align_corners=False, scale_factor given) on the 14x14 position grid ----
// (ATen upsample_bicubic2d: source index = scale * (dst + 0.5) - 0.5 with scale = 1 / scale_factor, NOT clamped; cubic
// convolution coefficients with A = -0.75; source taps clamped to the border.)
inline float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
inline float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
inline void cubic_coeffs(float t, float w[4]) {
  const float A = -0.75f;
  w[0] = cubic2(t + 1.f, A);
  w[1] = cubic1(t, A);
  w[2] = cubic1(1.f - t, A);
  w[3] = cubic2(2.f - t, A);
}
void resample_pos(const float* pos /*[197,384]*/, int gh, int gw, float* out /*[1+gh*gw,384]*/) {
  std::memcpy(out, pos, sizeof(float) * kVitDim);  // class position is kept
  // dino: scale_factor = ((h // 16 + 0.1) / 14, (w // 16 + 0.1) / 14), computed in double, handed to ATen as 1 / scale_factor
  const float sh = (float)(1.0 / (((double)gh + 0.1) / kVitGrid0)), sw = (float)(1.0 / (((double)gw + 0.1) / kVitGrid0));
  for (int oy = 0; oy < gh; ++oy) {
    const float ry = sh * ((float)oy + 0.5f) - 0.5f;
    const int iy = (int)std::floor(ry);
    float wy[4];
    cubic_coeffs(ry - (float)iy, wy);
    for (int ox = 0; ox < gw; ++ox) {
      const float rx = sw * ((float)ox + 0.5f) - 0.5f;
      const int ix = (int)std::floor(rx);
      float wx[4];
      cubic_coeffs(rx - (float)ix, wx);
      float* o = out + (size_t)(1 + oy * gw + ox) * kVitDim;
      for (int c = 0; c < kVitDim; ++c) o[c] = 0.f;
      for (int a = 0; a < 4; ++a) {
        const int y = std::min(std::max(iy - 1 + a, 0), kVitGrid0 - 1);
        for (int b = 0; b < 4; ++b) {
          const int x = std::min(std::max(ix - 1 + b, 0), kVitGrid0 - 1);
          const float w = wy[a] * wx[b];
          const float* src = pos + (size_t)(1 + y * kVitGrid0 + x) * kVitDim;
          for (int c = 0; c < kVitDim; ++c) o[c] += w * src[c];
        }
      }
    }
  }
}

// ---- one scale of the input pyramid ----
struct VitScale {
  int out_h, out_w;   // resized image
  int gh, gw;         // patch grid
  int tokens;         // 1 + gh * gw
  int row0;           // first activation row of this scale
  float inv_h, inv_w; // source-index scale (1 / scale_factor), unused when identity
  int identity;
  const float* pos;   // [tokens, 384]
};

// A[row, c*256 + ky*16 + kx] = resized normalised pixel of patch (py, px); class-token rows are zero.
// _resnet_normalize_image (image_feature_extractor.py:69) then F.interpolate(bilinear, align_corners=False, scale_factor) (:86).
__global__ void __launch_bounds__(256) vit_patchify_kernel(const float* __restrict__ img, int H, int W, VitScale sc, float* __restrict__ A) {
  const int tok = blockIdx.x, n = blockIdx.y;
  const int ky = threadIdx.x >> 4, kx = threadIdx.x & 15;
  float* row = A + (size_t)(sc.row0 + n * sc.tokens + tok) * kVitPatchK;
  if (tok == 0) {
    row[threadIdx.x] = 0.f;
    row[256 + threadIdx.x] = 0.f;
    row[512 + threadIdx.x] = 0.f;
    return;
  }
  const int p = tok - 1, py = p / sc.gw, px = p - py * sc.gw;
  const int oy = py * kVitPatch + ky, ox = px * kVitPatch + kx;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  int y0 = oy, y1 = oy, x0 = ox, x1 = ox;
  float ly = 0.f, lx = 0.f;
  if (!sc.identity) {
    float sy = sc.inv_h * ((float)oy + 0.5f) - 0.5f, sx = sc.inv_w * ((float)ox + 0.5f) - 0.5f;
    sy = fmaxf(sy, 0.f);
    sx = fmaxf(sx, 0.f);
    y0 = min((int)sy, H - 1);
    x0 = min((int)sx, W - 1);
    y1 = y0 + (y0 < H - 1 ? 1 : 0);
    x1 = x0 + (x0 < W - 1 ? 1 : 0);
    ly = sy - (float)y0;
    lx = sx - (float)x0;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* plane = img + ((size_t)n * 3 + c) * H * W;
    float v;
    if (sc.identity) {
      v = (plane[(size_t)oy * W + ox] - mean[c]) / stdv[c];
    } else {
      const float p00 = (plane[(size_t)y0 * W + x0] - mean[c]) / stdv[c], p01 = (plane[(size_t)y0 * W + x1] - mean[c]) / stdv[c];
      const float p10 = (plane[(size_t)y1 * W + x0] - mean[c]) / stdv[c], p11 = (plane[(size_t)y1 * W + x1] - mean[c]) / stdv[c];
      v = (1.f - ly) * ((1.f - lx) * p00 + lx * p01) + ly * ((1.f - lx) * p10 + lx * p11);
    }
    row[c * 256 + threadIdx.x] = v;
  }
}

// prepare_tokens: class row = cls_token + pos[0]; patch rows += pos[token]
__global__ void vit_pos_kernel(float* __restrict__ X, VitScale sc, int n_images, const float* __restrict__ cls) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = n_images * sc.tokens * (kVitDim / 4);
  if (idx >= total) return;
  const int c4 = idx % (kVitDim / 4), r = idx / (kVitDim / 4), tok = r % sc.tokens;
  float4* x = reinterpret_cast<float4*>(X + (size_t)(sc.row0 + r) * kVitDim) + c4;
  const float4 p = reinterpret_cast<const float4*>(sc.pos + (size_t)tok * kVitDim)[c4];
  float4 v = tok == 0 ? reinterpret_cast<const float4*>(cls)[c4] : *x;
  v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
  *x = v;
}

// per-row LayerNorm statistics of the residual stream (the affine part lives in the folded weights)
__global__ void vit_row_stats_kernel(const float* __restrict__ X, float* __restrict__ mean, float* __restrict__ rstd, int S) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= S) return;
  const float4* p = reinterpret_cast<const float4*>(X + (size_t)row * kVitDim);
  float4 v[3];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    v[i] = p[lane + 32 * i];
    sum += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float m = warp_sum(sum) * (1.0f / kVitDim);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float a = v[i].x - m, b = v[i].y - m, c = v[i].z - m, d = v[i].w - m;
    sq += a * a + b * b + c * c + d * d;
  }
  const float var = warp_sum(sq) * (1.0f / kVitDim);
  if (lane == 0) {
    mean[row] = m;
    rstd[row] = 1.0f / sqrtf(var + kVitLnEps);
  }
}

// Multi-head self-attention of one (image, scale) sequence of L <= 256 tokens, head width 64, on the warp-level tensor-core path
// (mma.sync m16n8k8 TF32, fp32 accumulate): the problem is 197 x 197 x 64 per head -- far below a 128-row wgmma tile pipeline's
// break-even -- so each warp owns 16 query rows end to end and the logits never leave registers:
//   S = (Q / 8) K^T   : A = Q fragments (registers, from global), B = K rows from shared memory (row stride 68 words: the 32
//                       lanes of a B-fragment load hit 32 distinct banks), in blocks of 8 key tiles (64 keys);
//   softmax            : online (running max / sum per query row, rescaling the output accumulator per key block); a query row
//                       lives in the 4 lanes of a quad -> two xor-shuffles per reduction;
//   O += P V           : the accumulator layout of S (row g: keys 2t, 2t+1) is reused directly as the A fragment of the second
//                       product by permuting the summation index (k-slot t <-> key 2t, k-slot t+4 <-> key 2t+1) and reading V rows
//                       in the same permuted order (again conflict-free with stride 68); no shuffles, no shared-memory round trip.
// CTA = (sequence, head, 128 query rows) = 8 warps; K and V of the head are staged once per CTA (TF32-rounded, zero padded).
// 64-key blocks keep the kernel at <= 128 registers: two CTAs = 16 warps per SM.  One launch covers every scale.
constexpr int kAttThreads = 256, kAttChunk = 128, kAttStride = 68, kAttKB = 8;
__host__ __device__ inline size_t vit_att_smem_bytes(int tiles) { return sizeof(uint32_t) * 2 * (size_t)tiles * 8 * kAttStride; }
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
struct VitAttArgs {  // one launch covers every scale: CTA ranges [block0[s], block0[s+1]) belong to scale s
  int n_scales;
  int max_tiles;  // key tiles of the longest sequence (shared-memory carve-up)
  int row0[kVitMaxScales], L[kVitMaxScales], chunks[kVitMaxScales], block0[kVitMaxScales + 1];
};
__global__ void __launch_bounds__(kAttThreads, 2) vit_attention_kernel(const float* __restrict__ qkv, float* __restrict__ att,
                                                                      const VitAttArgs A) {
  extern __shared__ __align__(16) uint32_t vsm[];
  uint32_t* Ks = vsm;                          // [tiles*8][68] TF32 bit patterns
  uint32_t* Vs = vsm + A.max_tiles * 8 * kAttStride;
  int sc = 0;
  while (sc + 1 < A.n_scales && (int)blockIdx.x >= A.block0[sc + 1]) ++sc;
  const int L = A.L[sc], chunks = A.chunks[sc], row0 = A.row0[sc];
  const int local = blockIdx.x - A.block0[sc];
  const int chunk = local % chunks, head = (local / chunks) % kVitHeads, seq = local / (chunks * kVitHeads);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int tiles = (L + 7) >> 3;  // key tiles of this scale
  const size_t base = (size_t)(row0 + seq * L) * (3 * kVitDim) + head * kVitHD;
  for (int idx = threadIdx.x; idx < tiles * 8 * (kVitHD / 4); idx += kAttThreads) {
    const int j = idx >> 4, c4 = idx & 15;
    float4 k4 = make_float4(0.f, 0.f, 0.f, 0.f), v4 = k4;
    if (j < L) {
      const float* src = qkv + base + (size_t)j * (3 * kVitDim) + c4 * 4;
      k4 = *reinterpret_cast<const float4*>(src + kVitDim);
      v4 = *reinterpret_cast<const float4*>(src + 2 * kVitDim);
    }
    *reinterpret_cast<uint4*>(Ks + j * kAttStride + c4 * 4) = make_uint4(to_tf32(k4.x), to_tf32(k4.y), to_tf32(k4.z), to_tf32(k4.w));
    *reinterpret_cast<uint4*>(Vs + j * kAttStride + c4 * 4) = make_uint4(to_tf32(v4.x), to_tf32(v4.y), to_tf32(v4.z), to_tf32(v4.w));
  }
  __syncthreads();
  const int r_base = chunk * kAttChunk + warp * 16;
  if (r_base >= L) return;  // whole warp; no block-level synchronisation follows
  const int ra = r_base + g, rb = r_base + g + 8;
  const float* qa = qkv + base + (size_t)min(ra, L - 1) * (3 * kVitDim);
  const float* qb = qkv + base + (size_t)min(rb, L - 1) * (3 * kVitDim);
  const float scale = 0.125f;  // head_dim ** -0.5, exact in TF32
  uint32_t q[kVitHD / 8][4];
#pragma unroll
  for (int ks = 0; ks < kVitHD / 8; ++ks) {
    q[ks][0] = to_tf32(qa[ks * 8 + t] * scale);
    q[ks][1] = to_tf32(qb[ks * 8 + t] * scale);
    q[ks][2] = to_tf32(qa[ks * 8 + t + 4] * scale);
    q[ks][3] = to_tf32(qb[ks * 8 + t + 4] * scale);
  }
  float o[kVitHD / 8][4];
#pragma unroll
  for (int dt = 0; dt < kVitHD / 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
  float ma = -INFINITY, mb = -INFINITY, la = 0.f, lb = 0.f;  // running max / (per-lane partial) sum of rows ra, rb
#pragma unroll 1
  for (int kb0 = 0; kb0 < tiles; kb0 += kAttKB) {  // block-uniform trip count; key kb0 * 8 < L is always valid
    float s[kAttKB][4];
#pragma unroll
    for (int nt = 0; nt < kAttKB; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      if (kb0 + nt < tiles) {
        const uint32_t* krow = Ks + ((kb0 + nt) * 8 + g) * kAttStride + t;
#pragma unroll
        for (int ks = 0; ks < kVitHD / 8; ++ks) mma_tf32(s[nt], q[ks], krow[ks * 8], krow[ks * 8 + 4]);
      }
    }
    // accumulator (g, 2t), (g, 2t+1) -> keys tile*8 + 2t, +1 of query row ra; (g+8, ..) -> the same keys of row rb
    float bma = -INFINITY, bmb = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < kAttKB; ++nt) {
      const int k0 = (kb0 + nt) * 8 + 2 * t;
      if (k0 >= L) s[nt][0] = s[nt][2] = -INFINITY;
      if (k0 + 1 >= L) s[nt][1] = s[nt][3] = -INFINITY;
      bma = fmaxf(bma, fmaxf(s[nt][0], s[nt][1]));
      bmb = fmaxf(bmb, fmaxf(s[nt][2], s[nt][3]));
    }
    bma = fmaxf(bma, __shfl_xor_sync(0xffffffffu, bma, 1));
    bma = fmaxf(bma, __shfl_xor_sync(0xffffffffu, bma, 2));
    bmb = fmaxf(bmb, __shfl_xor_sync(0xffffffffu, bmb, 1));
    bmb = fmaxf(bmb, __shfl_xor_sync(0xffffffffu, bmb, 2));
    const float na = fmaxf(ma, bma), nb = fmaxf(mb, bmb);            // finite: the block holds at least one valid key
    const float alpha_a = expf(ma - na), alpha_b = expf(mb - nb);    // first block: exp(-inf) = 0
    ma = na;
    mb = nb;
    float pa = 0.f, pb = 0.f;
#pragma unroll
    for (int nt = 0; nt < kAttKB; ++nt) {
      s[nt][0] = expf(s[nt][0] - ma);
      s[nt][1] = expf(s[nt][1] - ma);
      s[nt][2] = expf(s[nt][2] - mb);
      s[nt][3] = expf(s[nt][3] - mb);
      pa += s[nt][0] + s[nt][1];
      pb += s[nt][2] + s[nt][3];
    }
    la = la * alpha_a + pa;
    lb = lb * alpha_b + pb;
#pragma unroll
    for (int dt = 0; dt < kVitHD / 8; ++dt) {
      o[dt][0] *= alpha_a;
      o[dt][1] *= alpha_a;
      o[dt][2] *= alpha_b;
      o[dt][3] *= alpha_b;
    }
#pragma unroll
    for (int nt = 0; nt < kAttKB; ++nt) {
      if (kb0 + nt < tiles) {
        const uint32_t p[4] = {to_tf32(s[nt][0]), to_tf32(s[nt][2]), to_tf32(s[nt][1]), to_tf32(s[nt][3])};
        const uint32_t* v0 = Vs + ((kb0 + nt) * 8 + 2 * t) * kAttStride + g;
#pragma unroll
        for (int dt = 0; dt < kVitHD / 8; ++dt) mma_tf32(o[dt], p, v0[dt * 8], v0[kAttStride + dt * 8]);
      }
    }
  }
  la += __shfl_xor_sync(0xffffffffu, la, 1);
  la += __shfl_xor_sync(0xffffffffu, la, 2);
  lb += __shfl_xor_sync(0xffffffffu, lb, 1);
  lb += __shfl_xor_sync(0xffffffffu, lb, 2);
  const float ia = 1.0f / la, ib = 1.0f / lb;
  float* out = att + (size_t)(row0 + seq * L) * kVitDim + head * kVitHD + 2 * t;
#pragma unroll
  for (int dt = 0; dt < kVitHD / 8; ++dt) {
    if (ra < L) *reinterpret_cast<float2*>(out + (size_t)ra * kVitDim + dt * 8) = make_float2(o[dt][0] * ia, o[dt][1] * ia);
    if (rb < L) *reinterpret_cast<float2*>(out + (size_t)rb * kVitDim + dt * 8) = make_float2(o[dt][2] * ib, o[dt][3] * ib);
  }
}
// one launch for all scales; shared memory is sized by the longest sequence
int enqueue_vit_attention(Context* ctx, const float* qkv, float* att, const VitAttArgs& A, cudaStream_t st) {
  const size_t smem = vit_att_smem_bytes(A.max_tiles);
  if (ctx->attr_vit_att[0] < smem) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(vit_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ctx->attr_vit_att[0] = smem;
  }
  vit_attention_kernel<<<A.block0[A.n_scales], kAttThreads, smem, st>>>(qkv, att, A);
  return PDB_OK;
}

// z[n] = (1 / n_scales) * sum_scales LayerNorm(class row)  (vision_transformer forward: norm(x)[:, 0]; image_feature_extractor.py:74-83)
struct VitHeadArgs {
  int n_scales;
  int row0[kVitMaxScales];
  int tokens[kVitMaxScales];
};
__global__ void vit_head_kernel(const float* __restrict__ X, VitHeadArgs a, const float* __restrict__ gamma, const float* __restrict__ beta,
                                int n_images, float* __restrict__ z) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= n_images) return;
  float acc[kVitDim / 32];
#pragma unroll
  for (int i = 0; i < kVitDim / 32; ++i) acc[i] = 0.f;
  for (int s = 0; s < a.n_scales; ++s) {
    const float* x = X + (size_t)(a.row0[s] + n * a.tokens[s]) * kVitDim;
    float v[kVitDim / 32];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kVitDim / 32; ++i) {
      v[i] = x[lane + 32 * i];
      sum += v[i];
    }
    const float m = warp_sum(sum) * (1.0f / kVitDim);
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kVitDim / 32; ++i) sq += (v[i] - m) * (v[i] - m);
    const float rstd = 1.0f / sqrtf(warp_sum(sq) * (1.0f / kVitDim) + kVitLnEps);
#pragma unroll
    for (int i = 0; i < kVitDim / 32; ++i) {
      const int c = lane + 32 * i;
      const float y = (v[i] - m) * rstd * gamma[c] + beta[c];
      acc[i] = s == 0 ? y : acc[i] + y;
    }
  }
#pragma unroll
  for (int i = 0; i < kVitDim / 32; ++i) z[(size_t)n * kVitDim + lane + 32 * i] = acc[i] / (float)a.n_scales;
}

int vit_pos_table(Context* ctx, VitWeights* w, int gh, int gw, const float** out, cudaStream_t st) {
  if (gh == kVitGrid0 && gw == kVitGrid0) {
    *out = w->pos;
    return PDB_OK;
  }
  for (auto& e : w->pos_tables)
    if (std::get<0>(e) == gh && std::get<1>(e) == gw) {
      *out = std::get<2>(e);
      return PDB_OK;
    }
  const size_t n = (size_t)(1 + gh * gw) * kVitDim;
  std::vector<float> host(n);
  resample_pos(w->pos_host.data(), gh, gw, host.data());
  float* dev = nullptr;
  PDB_CUDA(ctx, cudaMalloc(&dev, n * sizeof(float)));
  PDB_CUDA(ctx, cudaMemcpyAsync(dev, host.data(), n * sizeof(float), cudaMemcpyHostToDevice, st));
  PDB_CUDA(ctx, cudaStreamSynchronize(st));  // `host` goes out of scope
  w->pos_tables.emplace_back(gh, gw, dev);
  *out = dev;
  return PDB_OK;
}

}  // namespace

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
  if (n_images < 1 || height < 1 || width < 1) return ctx->fail(PDB_ERR_INVALID, "bad image batch [%d,3,%d,%d]", n_images, height, width);
  if (n_scales < 1) return ctx->fail(PDB_ERR_INVALID, "scale_factors must not be empty");  // image_feature_extractor.py:75-76 (ValueError)
  if (n_scales > kVitMaxScales) return ctx->fail(PDB_ERR_LIMIT, "at most %d scale factors", kVitMaxScales);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  VitWeights* w = ctx->vit;

  VitScale sc[kVitMaxScales];
  VitHeadArgs head = {};
  head.n_scales = n_scales;
  long long rows = 0;
  for (int s = 0; s < n_scales; ++s) {
    const double f = scale_factors[s];
    if (!(f > 0.0)) return ctx->fail(PDB_ERR_INVALID, "scale factor %g", f);
    VitScale& v = sc[s];
    v.identity = f == 1.0;
    v.out_h = v.identity ? height : (int)std::floor((double)height * f);  // F.interpolate output size
    v.out_w = v.identity ? width : (int)std::floor((double)width * f);
    v.inv_h = v.inv_w = (float)(1.0 / f);
    v.gh = v.out_h / kVitPatch;
    v.gw = v.out_w / kVitPatch;
    if (v.gh < 1 || v.gw < 1) return ctx->fail(PDB_ERR_INVALID, "scale %g leaves a %dx%d image: smaller than one 16x16 patch", f, v.out_h, v.out_w);
    v.tokens = 1 + v.gh * v.gw;
    if (v.tokens > kVitMaxTokens)
      return ctx->fail(PDB_ERR_LIMIT, "%d tokens per image at scale %g (limit %d)", v.tokens, f, kVitMaxTokens);
    v.row0 = (int)rows;
    rows += (long long)n_images * v.tokens;
    if (int rc = vit_pos_table(ctx, w, v.gh, v.gw, &v.pos, st)) return rc;
    head.row0[s] = v.row0;
    head.tokens[s] = v.tokens;
  }
  if (rows > (1ll << 24)) return ctx->fail(PDB_ERR_LIMIT, "%lld tokens in one call", rows);
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

  VitAttArgs att_args = {};
  att_args.n_scales = n_scales;
  for (int s = 0; s < n_scales; ++s) {
    att_args.row0[s] = sc[s].row0;
    att_args.L[s] = sc[s].tokens;
    att_args.chunks[s] = (sc[s].tokens + kAttChunk - 1) / kAttChunk;
    att_args.max_tiles = std::max(att_args.max_tiles, (sc[s].tokens + 7) / 8);
    att_args.block0[s + 1] = att_args.block0[s] + n_images * kVitHeads * att_args.chunks[s];
  }
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
    if ((rc = enqueue_vit_attention(ctx, QKV, ATT, att_args, st))) break;
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
