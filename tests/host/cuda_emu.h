// TEST HARNESS (not product): a small CPU emulation of the CUDA execution model, enough to run the persistent
// cooperative kernels of posediffusion_b200/csrc UNMODIFIED on the host (tests/host/kernels_emu.cpp compiles csrc/ggs.cuh with
// g++ through this header).  It exists so that kernel variants written without GPU access can still be executed -- warp
// collectives, block barriers, shared memory, mbarrier / bulk-copy ring, grid-wide release / acquire barrier and all --
// against the CPU oracle.  It says nothing about performance and nothing about memory-model races.
//
// Model: one OS thread per CTA; inside it every CUDA thread is a ucontext coroutine, scheduled round-robin.  A coroutine
// runs until it reaches a rendezvous (`__syncthreads`, a `*_sync` warp collective, an mbarrier wait) and yields there until
// the rendezvous completes.  Static `__shared__` variables are `thread_local` (= per CTA, because all coroutines of a CTA
// live on one OS thread), dynamic shared memory is a per-CTA heap block; global memory is ordinary host memory, cross-CTA atomics are real atomics.
#pragma once
#include <cuda_runtime.h>  // vector types (float4, int4, dim3 ...) and empty __device__ / __global__ for a host compiler
#include <sched.h>
#include <ucontext.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#define PDB_EMU 1

// ---- storage classes ------------------------------------------------------------------------------------------
#undef __shared__
#define __shared__ thread_local
#undef __grid_constant__
#define __grid_constant__
#undef __launch_bounds__
#define __launch_bounds__(...)
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif

namespace emu {

constexpr int kWarp = 32;
constexpr size_t kStackBytes = 2048 * 1024;
constexpr size_t kSharedBytes = 232448;  // 227 KB opt-in maximum per CTA on sm_90

struct Cta {
  int nthreads = 0, nwarps = 0;
  std::vector<ucontext_t> ctx;
  std::vector<char*> stack;
  std::vector<char> done;
  ucontext_t sched;
  int current = -1, live = 0;
  // block barrier
  int block_count = 0;
  unsigned block_gen = 0;
  // warp rendezvous + exchange buffer
  std::vector<int> warp_count;
  std::vector<unsigned> warp_gen;
  std::vector<uint32_t> xch;  // [nwarps][32]
  std::function<void()> body;
  unsigned char* smem = nullptr;
};

extern thread_local Cta* g_cta;
extern thread_local uint3 g_threadIdx, g_blockIdx;
extern thread_local dim3 g_blockDim, g_gridDim;

inline void yield() { swapcontext(&g_cta->ctx[g_cta->current], &g_cta->sched); }

inline void block_barrier() {
  Cta* c = g_cta;
  const unsigned gen = c->block_gen;
  if (++c->block_count == c->live) {
    c->block_count = 0;
    c->block_gen++;
  } else {
    while (c->block_gen == gen) yield();
  }
}
inline void warp_barrier() {
  Cta* c = g_cta;
  const int w = c->current / kWarp;
  const unsigned gen = c->warp_gen[w];
  if (++c->warp_count[w] == kWarp) {  // kernels here always run whole warps with the full mask
    c->warp_count[w] = 0;
    c->warp_gen[w]++;
  } else {
    while (c->warp_gen[w] == gen) yield();
  }
}
inline uint32_t warp_exchange(uint32_t mine, int src_lane) {
  Cta* c = g_cta;
  const int w = c->current / kWarp, lane = c->current % kWarp;
  c->xch[w * kWarp + lane] = mine;
  warp_barrier();
  const uint32_t got = c->xch[w * kWarp + (src_lane & 31)];
  warp_barrier();
  return got;
}

// Run `body` as a grid of `grid` CTAs x `block` threads, all CTAs concurrently (cooperative launch semantics).
// Each CTA gets kSharedBytes of dynamic shared memory (Cta::smem; the kernels take it from there under PDB_EMU).
void launch(int grid, int block, const std::function<void()>& body);

}  // namespace emu

// ---- built-in variables ---------------------------------------------------------------------------------------
#define threadIdx (emu::g_threadIdx)
#define blockIdx (emu::g_blockIdx)
#define blockDim (emu::g_blockDim)
#define gridDim (emu::g_gridDim)

// ---- synchronisation and warp collectives ---------------------------------------------------------------------
inline void __syncthreads() { emu::block_barrier(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp_barrier(); }
template <typename T>
inline T __shfl_sync(unsigned, T v, int src) {
  static_assert(sizeof(T) == 4, "32-bit shuffles only");
  uint32_t bits;
  memcpy(&bits, &v, 4);
  bits = emu::warp_exchange(bits, src);
  memcpy(&v, &bits, 4);
  return v;
}
template <typename T>
inline T __shfl_xor_sync(unsigned m, T v, int lane_mask) {
  return __shfl_sync(m, v, (emu::g_cta->current % emu::kWarp) ^ lane_mask);
}
inline int __reduce_add_sync(unsigned m, int v) {
  int total = 0;
  for (int l = 0; l < 32; ++l) total += __shfl_sync(m, v, l);  // every lane makes the same 32 exchanges
  return total;
}

// ---- memory ---------------------------------------------------------------------------------------------------
template <typename T>
inline T __ldg(const T* p) { return *p; }
inline float __ldcg(const float* p) {
  uint32_t bits = __atomic_load_n(reinterpret_cast<const uint32_t*>(p), __ATOMIC_RELAXED);
  float v;
  memcpy(&v, &bits, 4);
  return v;
}
inline int __ldcg(const int* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
inline float4 __ldcg(const float4* p) { return *p; }
inline float atomicAdd(float* p, float v) {
  uint32_t* u = reinterpret_cast<uint32_t*>(p);
  uint32_t old = __atomic_load_n(u, __ATOMIC_RELAXED);
  for (;;) {
    float f;
    memcpy(&f, &old, 4);
    const float sum = f + v;
    uint32_t want;
    memcpy(&want, &sum, 4);
    if (__atomic_compare_exchange_n(u, &old, want, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return f;
  }
}
inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline int atomicOr(int* p, int v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
inline long long clock64() { return 0; }

// ---- arithmetic intrinsics ------------------------------------------------------------------------------------
inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
using std::max;
using std::min;

// ---- shared-state-space addresses, mbarrier, bulk copy (csrc/common.cuh uses these under PDB_EMU) ---------------
namespace emu {
inline uint32_t shared_addr(const void* p) { return (uint32_t)(reinterpret_cast<const unsigned char*>(p) - g_cta->smem) + 0x1000u; }
inline unsigned char* shared_ptr(uint32_t a) { return g_cta->smem + (a - 0x1000u); }
struct Mbar {  // 8 bytes, like the hardware object
  uint16_t phase, pending;  // current phase parity, arrivals still expected in this phase
  int32_t tx;               // bytes still expected in this phase
};
static_assert(sizeof(Mbar) == 8, "mbarrier object");
inline void mbar_check(Mbar* b, uint16_t count) {
  if (b->pending == 0 && b->tx == 0) {
    b->phase ^= 1;
    b->pending = count;
  }
}
// the expected arrival count is kept beside the barrier array by the user (always 1 in this code base)
inline void mbar_init(uint32_t bar, uint32_t count) {
  Mbar* b = reinterpret_cast<Mbar*>(shared_ptr(bar));
  if (count != 1) { fprintf(stderr, "emu: mbarrier count %u not supported\n", count); abort(); }
  b->phase = 0;
  b->pending = 1;
  b->tx = 0;
}
inline void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  Mbar* b = reinterpret_cast<Mbar*>(shared_ptr(bar));
  b->tx += (int32_t)bytes;
  b->pending -= 1;
  mbar_check(b, 1);
}
inline bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  Mbar* b = reinterpret_cast<Mbar*>(shared_ptr(bar));
  if (b->phase != parity) return true;  // the phase with this parity has completed
  yield();
  return false;
}
inline void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  if (bytes % 16 || dst % 16 || reinterpret_cast<uintptr_t>(src) % 16) { fprintf(stderr, "emu: misaligned bulk copy\n"); abort(); }
  if ((size_t)(dst - 0x1000u) + bytes > kSharedBytes) { fprintf(stderr, "emu: bulk copy past the end of shared memory\n"); abort(); }
  memcpy(shared_ptr(dst), src, bytes);
  Mbar* b = reinterpret_cast<Mbar*>(shared_ptr(bar));
  b->tx -= (int32_t)bytes;
  mbar_check(b, 1);
}
}  // namespace emu
