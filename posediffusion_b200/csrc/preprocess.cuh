// Image preprocessing of load_and_preprocess_images (util/load_img_folder.py): a centre-cropped uint8 HWC frame -> float32 CHW
// [3,S,S], i.e. uint8 -> fp32 (IEEE /255), bilinear resize (align_corners=False, no antialias) and transpose in one pass.
//
// Parity target: ATen's CPU upsample_bilinear2d.  scale = (float)in / (float)out; the source index is computed in double and
// rounded to float once; i1 = i0 + (i0 < in-1); out = l0h*(l0w*p00 + l1w*p01) + l1h*(l0w*p10 + l1w*p11), each product and sum
// rounded separately (no contraction into fma).  When in == out the weights are (1, 0) and the output is an exact copy.
//
// The host staging planner (csrc/api_pre.cu) and the kernel both take their rows from pre_tap(), so the rows uploaded are the
// rows read.  Only the rows some output row touches are staged, compacted in increasing order; the frame's staging region is
// [int2 rowmap[S]] (compact indices of i0 / i1 per output row) followed by the compact rows, each 3*side bytes (crop columns).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pdb {

struct PreTap {
  int i0, i1;
  float l0, l1;
};

// Source taps of destination index `dst` when `in` samples are resized to `out` (one axis).
__host__ __device__ inline PreTap pre_tap(int dst, int in, int out) {
  const float scale = (float)in / (float)out;
  const double s = (double)scale * ((double)dst + 0.5) - 0.5;
  const float src = (float)(s < 0.0 ? 0.0 : s);
  PreTap t;
  t.i0 = (int)src < in - 1 ? (int)src : in - 1;
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  float l1 = src - (float)t.i0;
  l1 = l1 < 0.f ? 0.f : (l1 > 1.f ? 1.f : l1);
  t.l1 = l1;
  t.l0 = 1.f - l1;
  return t;
}

// Round-to-nearest product / sum that nvcc may not fuse (the host compiler does not contract without -ffp-contract / FMA ISA).
__host__ __device__ inline float pre_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline float pre_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// Size of the row map at the start of a frame's staging region (keeps the rows 16-byte aligned).
__host__ __device__ inline size_t pre_map_bytes(int out) { return ((size_t)out * sizeof(int2) + 15) & ~(size_t)15; }

// Staging plan of one frame (host): marks the crop rows the S output rows touch, numbers them in increasing order and writes
// rowmap[S] (compact indices of each output row's two taps) and rows[count] (crop row of each compact row).  `compact` is
// scratch of `side` ints.  Returns the number of staged rows.
inline int pre_plan(int side, int S, int* compact, int2* rowmap, int* rows) {
  for (int r = 0; r < side; ++r) compact[r] = -1;
  for (int y = 0; y < S; ++y) {
    const PreTap t = pre_tap(y, side, S);
    compact[t.i0] = compact[t.i1] = 0;
  }
  int count = 0;
  for (int r = 0; r < side; ++r)
    if (compact[r] == 0) {
      rows[count] = r;
      compact[r] = count++;
    }
  for (int y = 0; y < S; ++y) {
    const PreTap t = pre_tap(y, side, S);
    rowmap[y] = make_int2(compact[t.i0], compact[t.i1]);
  }
  return count;
}

// One output pixel (x, y), all three channels.  `stage` is the frame's staging region, `out` its [3,S,S] output.
__host__ __device__ inline void pre_pixel(const uint8_t* stage, int side, int S, int x, int y, float* out) {
  const int2 rows = reinterpret_cast<const int2*>(stage)[y];
  const uint8_t* base = stage + pre_map_bytes(S);
  const size_t pitch = (size_t)3 * side;
  const PreTap th = pre_tap(y, side, S), tw = pre_tap(x, side, S);
  const uint8_t* r0 = base + (size_t)rows.x * pitch;
  const uint8_t* r1 = base + (size_t)rows.y * pitch;
  const size_t plane = (size_t)S * S, o = (size_t)y * S + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float p00 = (float)r0[tw.i0 * 3 + c] / 255.0f, p01 = (float)r0[tw.i1 * 3 + c] / 255.0f;
    const float p10 = (float)r1[tw.i0 * 3 + c] / 255.0f, p11 = (float)r1[tw.i1 * 3 + c] / 255.0f;
    const float top = pre_add(pre_mul(tw.l0, p00), pre_mul(tw.l1, p01));
    const float bot = pre_add(pre_mul(tw.l0, p10), pre_mul(tw.l1, p11));
    out[c * plane + o] = pre_add(pre_mul(th.l0, top), pre_mul(th.l1, bot));
  }
}

#ifdef __CUDACC__
__global__ void __launch_bounds__(256) preprocess_kernel(const uint8_t* __restrict__ stage, int side, int S, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * S) return;
  pre_pixel(stage, side, S, i % S, i / S, out);
}
#endif

}  // namespace pdb
