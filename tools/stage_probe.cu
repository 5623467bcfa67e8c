// Microbenchmark (GPU box only): cost of handing one activation tile from the CTAs that produce it to ALL persistent CTAs of a
// cooperative launch -- the step between two stages of the denoiser kernel (csrc/denoiser.cuh: 43 such hand-overs per
// diffusion step).  A tile is ROWS x K floats; P producer CTAs write 8 features x ROWS tokens each (K = 8 P), then every
// CTA needs the whole tile in shared memory before it can start its next item.
//
//   mode 0  plain stores, group barrier (__syncthreads, red.release.gpu, acquire poll, __syncthreads), then ONE round of
//           float4 loads of the tile -- what the kernel does
//   mode 1  flag-carrying words: every value is published as one 64-bit {fp32, tag} store (st.relaxed.gpu.b64, single-copy
//           atomic), consumers load the tile as 2 x 64-bit vectors and re-load the words whose tag is not there yet;
//           no barrier, no fence
//   mode 2  mode 1, but consumers first poll ONE word per producer (its last store) and only then read the tile once
//           (re-loading stragglers); less polling traffic
//
// CTAs that produce nothing can fall behind the producers by more than the 4 rotating buffers; the probe therefore accepts
// NEWER tags as well (the kernel cannot: there every reader of a buffer is, transitively, a dependency of its next writer).
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a tools/stage_probe.cu -o build/stage_probe
//   build/stage_probe [rows=20] [producers=64] [iters=20000]
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

constexpr int kThreads = 256;
constexpr int kBufs = 4;

__device__ __forceinline__ void st_ll(unsigned long long* p, float v, unsigned tag) {
  const unsigned long long w = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ void ld_ll2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.b64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ unsigned long long ld_ll(const unsigned long long* p) {
  unsigned long long w;
  asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
  return w;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add_u32(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// PAIRS = 16-byte loads per thread that cover the tile (ROWS * K / 2 words / 256 threads, rounded up)
template <int MODE, int PAIRS>
__global__ void __launch_bounds__(kThreads, 1)
probe(float* plain, unsigned long long* ll, unsigned* bar, int rows, int producers, int iters, float* out, long long* cycles) {
  extern __shared__ __align__(16) float tile[];
  const int K = producers * 8;
  const int words = rows * K;
  const int G = gridDim.x;
  float v = (float)(blockIdx.x + 1) * 1e-3f;
  unsigned count = 0;
  const long long c0 = clock64();
  for (int it = 0; it < iters; ++it) {
    const unsigned tag = (unsigned)it + 1u;
    float* pb = plain + (size_t)(it % kBufs) * words;
    unsigned long long* lb = ll + (size_t)(it % kBufs) * words;
    // ---- produce: thread (token s, feature f) of producer CTA c ----
    const int s = threadIdx.x >> 3, f = threadIdx.x & 7;
    if ((int)blockIdx.x < producers && s < rows) {
      const int e = s * K + blockIdx.x * 8 + f;
      if (MODE == 0) pb[e] = v;
      else st_ll(lb + e, v, tag);
    }
    // ---- hand over ----
    if (MODE == 0) {
      ++count;
      __syncthreads();
      if (threadIdx.x == 0) {
        red_release_add_u32(bar, 1u);
        while (ld_acquire_u32(bar) < count * (unsigned)G) {
        }
      }
      __syncthreads();
      float4 r[PAIRS / 2 + 1];
#pragma unroll
      for (int i = 0; i < (PAIRS + 1) / 2; ++i) {
        const int idx = threadIdx.x + i * kThreads;
        r[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (idx * 4 < words) r[i] = __ldcg(reinterpret_cast<const float4*>(pb) + idx);
      }
#pragma unroll
      for (int i = 0; i < (PAIRS + 1) / 2; ++i) {
        const int idx = threadIdx.x + i * kThreads;
        if (idx * 4 < words) reinterpret_cast<float4*>(tile)[idx] = r[i];
      }
    } else {
      if (MODE == 2) {  // one canary per producer: its last feature of the last token
        for (int p = threadIdx.x; p < producers; p += kThreads) {
          const unsigned long long* w = lb + (size_t)(rows - 1) * K + p * 8 + 7;
          while ((int)((unsigned)(ld_ll(w) >> 32) - tag) < 0) {
          }
        }
        __syncthreads();
      }
      unsigned long long a[PAIRS], b[PAIRS];
#pragma unroll
      for (int i = 0; i < PAIRS; ++i) {
        const int idx = threadIdx.x + i * kThreads;
        a[i] = b[i] = (unsigned long long)tag << 32;
        if (idx * 2 < words) ld_ll2(lb + 2 * idx, a[i], b[i]);
      }
#pragma unroll
      for (int i = 0; i < PAIRS; ++i) {
        const int idx = threadIdx.x + i * kThreads;
        if (idx * 2 < words) {
          while ((int)((unsigned)(a[i] >> 32) - tag) < 0 || (int)((unsigned)(b[i] >> 32) - tag) < 0) ld_ll2(lb + 2 * idx, a[i], b[i]);
          reinterpret_cast<float2*>(tile)[idx] = make_float2(__uint_as_float((unsigned)a[i]), __uint_as_float((unsigned)b[i]));
        }
      }
    }
    __syncthreads();
    // ---- "item": every CTA's next value depends on the whole tile having arrived ----
    v = tile[(threadIdx.x * 37 + it) % words] * 0.5f + tile[(threadIdx.x * 11 + 3 * it) % words] * 0.25f + 1e-3f;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    cycles[blockIdx.x] = clock64() - c0;
    out[blockIdx.x] = v;
  }
}

template <int MODE, int PAIRS>
static void run(const char* name, int rows, int producers, int iters, int grid) {
  const int K = producers * 8, words = rows * K;
  float* plain;
  unsigned long long* ll;
  unsigned* bar;
  float* out;
  long long* cycles;
  CK(cudaMalloc(&plain, sizeof(float) * words * kBufs));
  CK(cudaMalloc(&ll, sizeof(unsigned long long) * words * kBufs));
  CK(cudaMalloc(&bar, 256));
  CK(cudaMalloc(&out, sizeof(float) * grid));
  CK(cudaMalloc(&cycles, sizeof(long long) * grid));
  const size_t smem = sizeof(float) * words + 64;
  CK(cudaFuncSetAttribute(probe<MODE, PAIRS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  float best = 1e30f;
  for (int rep = 0; rep < 3; ++rep) {
    CK(cudaMemset(plain, 0, sizeof(float) * words * kBufs));
    CK(cudaMemset(ll, 0, sizeof(unsigned long long) * words * kBufs));
    CK(cudaMemset(bar, 0, 256));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    void* args[] = {&plain, &ll, &bar, &rows, &producers, &iters, &out, &cycles};
    CK(cudaEventRecord(e0));
    CK(cudaLaunchCooperativeKernel((void*)probe<MODE, PAIRS>, dim3(grid), dim3(kThreads), args, smem, 0));
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  std::vector<float> h(grid);
  CK(cudaMemcpy(h.data(), out, sizeof(float) * grid, cudaMemcpyDeviceToHost));
  bool same = true;  // every CTA computed from the same tile -> CTAs with equal thread-0 inputs agree; just report a checksum
  double sum = 0;
  for (float x : h) sum += x;
  (void)same;
  printf("%-34s rows %3d K %4d (%6.1f KB%s): %7.3f us per hand-over   checksum %.6f\n", name, rows, K,
         words * (MODE == 0 ? 4 : 8) / 1024.0, MODE == 0 ? "" : " flagged", best * 1e3f / iters, sum);
  CK(cudaFree(plain));
  CK(cudaFree(ll));
  CK(cudaFree(bar));
  CK(cudaFree(out));
  CK(cudaFree(cycles));
}

template <int PAIRS>
static void run_all(int rows, int producers, int iters, int grid) {
  run<0, PAIRS>("barrier + plain tile load", rows, producers, iters, grid);
  run<1, PAIRS>("flagged words, poll the tile", rows, producers, iters, grid);
  run<2, PAIRS>("flagged words, canaries first", rows, producers, iters, grid);
}

int main(int argc, char** argv) {
  int rows = argc > 1 ? atoi(argv[1]) : 20;
  int producers = argc > 2 ? atoi(argv[2]) : 64;
  int iters = argc > 3 ? atoi(argv[3]) : 20000;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int grid = prop.multiProcessorCount;
  if (producers > grid) producers = grid;
  const int words = rows * producers * 8;
  const int pairs = (words / 2 + kThreads - 1) / kThreads;
  printf("%s, %d CTAs x %d threads, %d producers, tile %d x %d\n", prop.name, grid, kThreads, producers, rows, producers * 8);
  if (pairs <= 8) run_all<8>(rows, producers, iters, grid);
  else if (pairs <= 20) run_all<20>(rows, producers, iters, grid);
  else if (pairs <= 40) run_all<40>(rows, producers, iters, grid);
  else printf("tile too large for this probe (%d pairs per thread)\n", pairs);
  return 0;
}
