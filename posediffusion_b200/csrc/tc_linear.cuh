// Tensor-core linear layer for the batched denoiser (S = B*N >= 128 tokens per GPU, BASELINE config 4) and the ViT backbone:
//   Y[S, O] = epilogue( X[S, K] @ W[O, K]^T )
// as Hopper warpgroup MMA tiles fed by TMA, written directly in PTX for sm_90a:
//   * TMA (`cp.async.bulk.tensor.2d`) stages 128-row x 32-float (128 B, SWIZZLE_128B) boxes of the M-side operand and
//     BN-row boxes of the N-side operand into a shared-memory ring, completion counted on mbarriers;
//   * two consumer warpgroups each issue `wgmma.mma_async.m64nBNk8.f32.tf32.tf32` (fp32 operands read as TF32, fp32
//     accumulate) on 64 of the tile's 128 M-side rows, both operands read from shared memory through descriptors, 4 K-steps of
//     8 per stage; the 64 x BN fp32 accumulator of a warpgroup lives in its registers (BN / 2 per thread);
//   * the kernel is persistent over output tiles; one wgmma group stays in flight while the previous stage is released, and
//     the producer keeps filling the ring for the next tile while the consumers run the epilogue (bias / folded LayerNorm /
//     residual / ReLU / GELU) from registers straight to global memory.
// Warp roles: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = MMA + epilogue (M-side rows 0-63 and 64-127).
//
// Swap-AB instantiation (kSwap, few tokens: S <= 96): the WEIGHTS take the 128-row M side (A = 128 features x 32 k) and
// the tokens the N side (B = BN tokens x 32 k, BN = 32 / 64 / 96, rows beyond S zero-filled by TMA), i.e. the tile computes
// Y^T[128 features, BN tokens].  No tensor-core work is spent on padding tokens up to 128 rows.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace pdb {

constexpr int kTcThreads = 384;
constexpr int kTcStages = 4;  // default ring depth (64-feature tiles: two CTAs share an SM)
constexpr int kTcBM = 128;  // M-side rows per tile (two warpgroups x wgmma M = 64)
constexpr int kTcBK = 32;   // floats per stage (128 bytes = one swizzle atom), 4 wgmma K-steps of 8
constexpr int kTcConsumerWarps = 8;

struct TcEpilogue {
  const float* bias;      // [O] or null
  const int* t_ptr;       // optional: device-side timestep; the bias row used is bias + (*t_ptr) * bias_t_stride
  int bias_t_stride;
  const float* residual;  // [S, ldr] or null (may alias Y: each element is read then written by the same thread)
  int ldr;
  const float* row_mean;  // folded LayerNorm: Y = rstd_s * (acc - mean_s * colsum_o) + bias_o   (all three or none)
  const float* row_rstd;
  const float* colsum;
  float* Y;
  int ldy;
  int S, O, K;
  int relu;
  int gelu;  // exact (erf) GELU, torch.nn.functional.gelu default
  int pdl;          // launch with programmatic stream serialization (the kernel's prologue overlaps the previous kernel's tail)
  int allow_small;  // caller opts in to the small-problem regime below (split-K sums in arrival order: not bit-reproducible)
  // Small problems (fewer tiles than SMs), set by the launcher:
  int splits;  // split-K factor (>= 1).  > 1: Y already holds the residual (in-place residual stream); every split adds its
               // partial product to it with vector reductions (red.global.add.v2.f32), split 0 also the bias.
  int stats;   // 1: the folded-LayerNorm row statistics are computed inside the kernel, by the consumer warpgroups, from the X
               // operand tiles as they pass through shared memory (row_mean / row_rstd are not read); needs splits == 1
};

__host__ __device__ inline size_t tc_smem_bytes(int BN, int stages = kTcStages) {
  return (size_t)stages * (kTcBM * 128 + BN * 128) + 256 + 1024;  // ring + barriers + alignment slack
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(map), "r"(bar), "r"(c0), "r"(c1)
               : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma): start address >> 4 (bits 0-13), LBO unused (1),
// SBO = 8 rows x 128 B = 1024 B between core-matrix groups (bits 32-45), base offset 0 (every tile is 1024-byte aligned),
// layout type 1 = SWIZZLE_128B (bits 62-63).
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, TF32 products, fp32 accumulate; `accumulate` == 0 overwrites D.  Accumulator
// fragment of thread t of the warpgroup: d[4i + 2h + e] = D[16 (t / 32) + (t % 32) / 4 + 8h][8i + 2 (t % 4) + e].
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[48], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
      "%48, %49, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

// Persistent: every CTA walks the work list (work = blockIdx.x, + gridDim.x, ...; work = split * tiles + tile, N-side tile index
// fastest so that CTAs running side by side share the same 128 M-side rows in L2; split s of E.splits covers the k-blocks
// [s, s+1) * K/32 / splits).  The ring is shared by the two consumer warpgroups: a stage is released once all 8 consumer
// warps have retired the MMAs that read it (and, with E.stats, read its X rows).
template <int BN, int ST = kTcStages, bool kSwap = false>
__global__ void __launch_bounds__(kTcThreads, 1)
tc_linear_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const TcEpilogue E) {
  static_assert(kSwap ? (BN == 32 || BN == 64 || BN == 96) : (BN == 64 || BN == 128), "N-side tile");
  extern __shared__ unsigned char tc_smem_raw[];
  const uint32_t raw = smem_u32(tc_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024-byte alignment
  constexpr uint32_t kABytes = kTcBM * 128, kBBytes = BN * 128, kStageBytes = kABytes + kBBytes;
  const uint32_t bar_base = base + ST * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + s * 8; };
  auto empty_bar = [&](int s) { return bar_base + (ST + s) * 8; };

  pdl_trigger();  // the next kernel of a programmatic chain may start its own prologue now (it still waits for our completion)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = E.K / kTcBK;
  // tile list: the N-side index runs fastest.  normal: M side = 128 tokens, N side = BN features; swap: M side = 128 features,
  // N side = BN tokens.  (m0, n0) below are always (M-side offset, N-side offset).
  const int n_tiles = kSwap ? (E.S + BN - 1) / BN : E.O / BN;
  const int total_tiles = n_tiles * (kSwap ? E.O / kTcBM : (E.S + kTcBM - 1) / kTcBM);
  const int splits = kSwap ? 1 : (E.splits > 1 ? E.splits : 1);
  const int total_work = total_tiles * splits;
  const bool stats = !kSwap && E.stats && splits == 1;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    for (int s = 0; s < ST; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), kTcConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touched only this CTA's shared memory; global reads and writes start below

  if (warp < 4) {
    if (threadIdx.x == 0) {  // ===== TMA producer =====
      int it = 0;
      for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
        const int tile = work % total_tiles, split = work / total_tiles;
        const int m0 = (tile / n_tiles) * kTcBM, n0 = (tile % n_tiles) * BN;
        const int kb0 = split * num_kb / splits, kb1 = (split + 1) * num_kb / splits;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % ST;
          const uint32_t ph = (it / ST) & 1;
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_arrive_expect_tx(full_bar(s), kStageBytes);
          tma_load_2d(base + s * kStageBytes, kSwap ? &map_w : &map_x, kb * kTcBK, m0, full_bar(s));
          tma_load_2d(base + s * kStageBytes + kABytes, kSwap ? &map_x : &map_w, kb * kTcBK, n0, full_bar(s));
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns M-side rows [64 wg, 64 wg + 64) of every tile =====
  const int wg = (warp >> 2) - 1, wq = warp & 3, t = threadIdx.x & 127;
  const int q2 = 2 * (lane & 3);
  const float* bias = E.bias;
  if (bias && E.t_ptr) bias += (size_t)(*E.t_ptr) * E.bias_t_stride;
  float acc[BN / 2] = {};
  int it = 0;
  for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
    const int tile = work % total_tiles, split = work / total_tiles;
    const int m0 = (tile / n_tiles) * kTcBM, n0 = (tile % n_tiles) * BN;
    const int kb0 = split * num_kb / splits, kb1 = (split + 1) * num_kb / splits;
    // folded-LayerNorm statistics (stats): thread t sums half t & 1 of row t >> 1 of this warpgroup's 64 X rows.  A row is 128
    // contiguous bytes of a stage (SWIZZLE_128B only permutes the 16-byte chunks inside it, and a sum does not care); the
    // chunk order is rotated by row so that a warp's loads spread over all banks.  Shifted by the first value stored in the
    // row, which both halves read (one-pass variance without cancellation).
    float pivot = 0.f, s1 = 0.f, s2 = 0.f;
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const int s = it % ST;
      mbar_wait(full_bar(s), (it / ST) & 1);
      const uint32_t a_tile = base + s * kStageBytes + (uint32_t)wg * (64 * 128);
      const uint64_t da = wgmma_desc_k128(a_tile);
      const uint64_t db = wgmma_desc_k128(base + s * kStageBytes + kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTcBK / 8; ++k)  // advance 8 floats = 32 bytes inside the swizzle atom: +2 in the (>>4) address field
        wgmma_tf32(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb > kb0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      if (stats) {
        const uint32_t rowaddr = a_tile + (uint32_t)(t >> 1) * 128u;
        if (kb == kb0) pivot = lds_f4(rowaddr).x;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 x = lds_f4(rowaddr + (uint32_t)((((t & 1) << 2) | ((j + (t >> 1)) & 3)) << 4));
          const float a = x.x - pivot, b = x.y - pivot, c = x.z - pivot, d = x.w - pivot;
          s1 += (a + b) + (c + d);
          s2 += (a * a + b * b) + (c * c + d * d);
        }
      }
      wgmma_wait<1>();  // the MMAs of the previous stage have retired: hand that stage back to the producer
      if (kb > kb0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar((it + ST - 1) % ST));
      }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar((it + ST - 1) % ST));

    float st_mean = 0.f, st_rstd = 1.f;  // statistics of row t >> 1 (both threads of the row hold them)
    if (stats) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
      const float inv_k = 1.0f / (float)E.K;
      const float m = s1 * inv_k;
      st_mean = pivot + m;
      st_rstd = 1.0f / sqrtf(fmaxf(s2 * inv_k - m * m, 0.f) + 1e-5f);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int fr = 16 * wq + (lane >> 2) + 8 * h;  // fragment row inside the warpgroup's 64 rows
      if constexpr (kSwap) {
        // fragment row = feature o, column = token: 8 lanes store 8 consecutive features of a token (one 32-byte sector)
        const int o = m0 + 64 * wg + fr;
        const float b_o = bias ? __ldg(bias + o) : 0.f;
        const float cs_o = E.colsum ? __ldg(E.colsum + o) : 0.f;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int srow = n0 + 8 * i + q2 + e;
            if (srow < E.S) {
              float x = acc[4 * i + 2 * h + e];
              if (E.colsum) x = __ldg(E.row_rstd + srow) * (x - __ldg(E.row_mean + srow) * cs_o);
              x += b_o;
              if (E.residual) x += E.residual[(size_t)srow * E.ldr + o];
              if (E.relu) x = fmaxf(x, 0.f);
              if (E.gelu) x = 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
              E.Y[(size_t)srow * E.ldy + o] = x;
            }
          }
        }
      } else {
        // fragment row = token, columns = features: the 4 lanes of a quad store 8 consecutive features (one 32-byte sector)
        const int row = m0 + 64 * wg + fr;
        float mean = 0.f, rstd = 1.f;
        if (stats) {  // the row's statistics live with thread 2 fr of this warpgroup: lane 2 fr % 32 of this warp
          mean = __shfl_sync(0xffffffffu, st_mean, (2 * fr) & 31);
          rstd = __shfl_sync(0xffffffffu, st_rstd, (2 * fr) & 31);
        } else if (E.colsum && row < E.S) {
          mean = E.row_mean[row];
          rstd = E.row_rstd[row];
        }
        if (row < E.S) {
          float* yrow = E.Y + (size_t)row * E.ldy + n0 + q2;
          const float* rrow = E.residual ? E.residual + (size_t)row * E.ldr + n0 + q2 : nullptr;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            const int col = n0 + 8 * i + q2;
            float o0 = acc[4 * i + 2 * h], o1 = acc[4 * i + 2 * h + 1];
            if (E.colsum) {
              o0 = rstd * (o0 - mean * __ldg(E.colsum + col));
              o1 = rstd * (o1 - mean * __ldg(E.colsum + col + 1));
            }
            if (bias && split == 0) {
              o0 += __ldg(bias + col);
              o1 += __ldg(bias + col + 1);
            }
            if (splits > 1) {  // Y holds the residual already: accumulate this split's partial product on top of it
              red_add_v2(yrow + 8 * i, o0, o1);
              continue;
            }
            if (rrow) {
              const float2 r = *reinterpret_cast<const float2*>(rrow + 8 * i);
              o0 += r.x;
              o1 += r.y;
            }
            if (E.relu) {
              o0 = fmaxf(o0, 0.f);
              o1 = fmaxf(o1, 0.f);
            }
            if (E.gelu) {
              o0 = 0.5f * o0 * (1.0f + erff(o0 * 0.70710678118654752f));
              o1 = 0.5f * o1 * (1.0f + erff(o1 * 0.70710678118654752f));
            }
            *reinterpret_cast<float2*>(yrow + 8 * i) = make_float2(o0, o1);
          }
        }
      }
    }
  }
}

struct Context;
// Y = epilogue(X[S,K] @ W[O,K]^T) on the tensor cores (csrc/api_tc.cu).  K % 32 == 0, O % 64 == 0, 16-byte aligned pointers.
int enqueue_tc_linear(Context* ctx, const float* X, const float* W, TcEpilogue E, cudaStream_t st);
// true when the launcher will treat (S, O) as a small problem: 8-deep ring, split-K for in-place residual GEMMs, and in-kernel
// LayerNorm statistics when E.stats is set (the caller then skips its row-statistics kernel)
bool tc_linear_small(const Context* ctx, int S, int O);

}  // namespace pdb
