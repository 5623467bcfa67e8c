// DINO ViT-S/16 pieces shared by the inference path (csrc/api_vit.cu) and the training path (csrc/api_vit_train.cu): the
// architecture constants, the input pyramid's geometry, patchify / position kernels, the tensor-core attention forward, the head,
// and the bicubic resampling of the position table.  Everything with a definition lives in an anonymous namespace, so each
// translation unit that includes this header owns its copy of the kernels.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <tuple>
#include <vector>

#include "context.cuh"
#include "tc_linear.cuh"

namespace pdb {

constexpr int kVitDim = 384, kVitHeads = 6, kVitHD = 64, kVitDepth = 12, kVitMlp = 1536, kVitPatch = 16;
constexpr int kVitPatchK = 3 * kVitPatch * kVitPatch;  // 768
constexpr int kVitGrid0 = 14;                          // native 224 / 16 position grid
constexpr int kVitMaxTokens = 256;                     // tokens per (image, scale) the attention kernel keeps in shared memory
constexpr int kVitMaxScales = 4;
constexpr int kVitMaxImages = 65535;                   // vit_patchify_kernel puts the image index on gridDim.y
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
using namespace pdb;

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
// The resampling as a sparse linear map R: patch o of the gh x gw grid reads 16 cells of the stored 14x14 grid, taps
// (cell[16 o + k], weight[16 o + k]) in row-major (a, b) order.  resample_pos applies R on the host; the training path applies R
// and its adjoint on the device (csrc/vit_train.cuh).
constexpr int kVitPosTaps = 16;
void pos_taps(int gh, int gw, int* cell /*[gh*gw*16]*/, float* weight /*[gh*gw*16]*/) {
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
      const size_t o = (size_t)(oy * gw + ox) * kVitPosTaps;
      for (int a = 0; a < 4; ++a) {
        const int y = std::min(std::max(iy - 1 + a, 0), kVitGrid0 - 1);
        for (int b = 0; b < 4; ++b) {
          const int x = std::min(std::max(ix - 1 + b, 0), kVitGrid0 - 1);
          cell[o + a * 4 + b] = y * kVitGrid0 + x;
          weight[o + a * 4 + b] = wy[a] * wx[b];
        }
      }
    }
  }
}
void resample_pos(const float* pos /*[197,384]*/, int gh, int gw, float* out /*[1+gh*gw,384]*/) {
  std::memcpy(out, pos, sizeof(float) * kVitDim);  // class position is kept
  std::vector<int> cell((size_t)gh * gw * kVitPosTaps);
  std::vector<float> weight(cell.size());
  pos_taps(gh, gw, cell.data(), weight.data());
  for (int p = 0; p < gh * gw; ++p) {
    float* o = out + (size_t)(1 + p) * kVitDim;
    for (int c = 0; c < kVitDim; ++c) o[c] = 0.f;
    for (int k = 0; k < kVitPosTaps; ++k) {
      const float w = weight[(size_t)p * kVitPosTaps + k];
      const float* src = pos + (size_t)(1 + cell[(size_t)p * kVitPosTaps + k]) * kVitDim;
      for (int c = 0; c < kVitDim; ++c) o[c] += w * src[c];
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

// The pyramid of one call: per scale the resized size (F.interpolate's floor(size * f)), its patch grid and its first activation
// row (scale-major, then image, then token).  Returns PDB_OK or the error code with the reason in `why`; launches nothing.
int vit_plan_scales(int n_images, int height, int width, const double* scale_factors, int n_scales, VitScale* sc, long long* rows_out,
                    char* why, size_t why_len) {
  if (n_images < 1 || height < 1 || width < 1) {
    snprintf(why, why_len, "bad image batch [%d,3,%d,%d]", n_images, height, width);
    return PDB_ERR_INVALID;
  }
  if (n_images > kVitMaxImages) {
    snprintf(why, why_len, "%d images in one call (limit %d)", n_images, kVitMaxImages);
    return PDB_ERR_LIMIT;
  }
  if (n_scales < 1) {  // image_feature_extractor.py:75-76 (ValueError)
    snprintf(why, why_len, "scale_factors must not be empty");
    return PDB_ERR_INVALID;
  }
  if (n_scales > kVitMaxScales) {
    snprintf(why, why_len, "at most %d scale factors", kVitMaxScales);
    return PDB_ERR_LIMIT;
  }
  long long rows = 0;
  for (int s = 0; s < n_scales; ++s) {
    const double f = scale_factors[s];
    if (!(f > 0.0)) {
      snprintf(why, why_len, "scale factor %g", f);
      return PDB_ERR_INVALID;
    }
    VitScale& v = sc[s];
    v.identity = f == 1.0;
    v.out_h = v.identity ? height : (int)std::floor((double)height * f);  // F.interpolate output size
    v.out_w = v.identity ? width : (int)std::floor((double)width * f);
    v.inv_h = v.inv_w = (float)(1.0 / f);
    v.gh = v.out_h / kVitPatch;
    v.gw = v.out_w / kVitPatch;
    if (v.gh < 1 || v.gw < 1) {
      snprintf(why, why_len, "scale %g leaves a %dx%d image: smaller than one 16x16 patch", f, v.out_h, v.out_w);
      return PDB_ERR_INVALID;
    }
    v.tokens = 1 + v.gh * v.gw;
    if (v.tokens > kVitMaxTokens) {
      snprintf(why, why_len, "%d tokens per image at scale %g (limit %d)", v.tokens, f, kVitMaxTokens);
      return PDB_ERR_LIMIT;
    }
    v.row0 = (int)rows;
    v.pos = nullptr;
    rows += (long long)n_images * v.tokens;
  }
  if (rows > (1ll << 24)) {
    snprintf(why, why_len, "%lld tokens in one call", rows);
    return PDB_ERR_LIMIT;
  }
  *rows_out = rows;
  return PDB_OK;
}

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
// `attr` is the including translation unit's slot of Context::attr_vit_att (each owns its copy of the kernel)
int enqueue_vit_attention(Context* ctx, const float* qkv, float* att, const VitAttArgs& A, size_t& attr, cudaStream_t st) {
  const size_t smem = vit_att_smem_bytes(A.max_tiles);
  if (attr < smem) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(vit_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  vit_attention_kernel<<<A.block0[A.n_scales], kAttThreads, smem, st>>>(qkv, att, A);
  return PDB_OK;
}

VitAttArgs vit_att_args(const VitScale* sc, int n_scales, int n_images) {
  VitAttArgs a = {};
  a.n_scales = n_scales;
  for (int s = 0; s < n_scales; ++s) {
    a.row0[s] = sc[s].row0;
    a.L[s] = sc[s].tokens;
    a.chunks[s] = (sc[s].tokens + kAttChunk - 1) / kAttChunk;
    a.max_tiles = std::max(a.max_tiles, (sc[s].tokens + 7) / 8);
    a.block0[s + 1] = a.block0[s] + n_images * kVitHeads * a.chunks[s];
  }
  return a;
}

// z[n] = (1 / n_scales) * sum_scales LayerNorm(class row)  (vision_transformer forward: norm(x)[:, 0]; image_feature_extractor.py:74-83)
struct VitHeadArgs {
  int n_scales;
  int row0[kVitMaxScales];
  int tokens[kVitMaxScales];
};
VitHeadArgs vit_head_args(const VitScale* sc, int n_scales) {
  VitHeadArgs h = {};
  h.n_scales = n_scales;
  for (int s = 0; s < n_scales; ++s) {
    h.row0[s] = sc[s].row0;
    h.tokens[s] = sc[s].tokens;
  }
  return h;
}
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

// dino's interpolate_pos_encoding keeps the stored table only for 196 patches of a SQUARE image (it compares pixel sizes), so a
// 224x232 input resamples the 14x14 grid with scale 14.1 / 14; that resampled 14x14 table is cached in pos_tables like any other.
int vit_pos_table(Context* ctx, VitWeights* w, int gh, int gw, bool square, const float** out, cudaStream_t st) {
  if (gh == kVitGrid0 && gw == kVitGrid0 && square) {
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
