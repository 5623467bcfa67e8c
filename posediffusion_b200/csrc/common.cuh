// Shared device/host helpers for the posediff_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pdb {

constexpr int kTargetDim = 9;
constexpr int kMaxFrames = 128;

// ---------------------------------------------------------------------------------------------
// Warp helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Reduce 16 per-lane values across the 32 lanes of a warp with 16 shuffles (instead of 80):
// at every butterfly step each lane hands half of its slots to its partner.  On return lane L
// (both lanes of a pair L, L^1 hold the same value) owns slot  ((L>>4)&1)*8 + ((L>>3)&1)*4 +
// ((L>>2)&1)*2 + ((L>>1)&1)  in v[0].  Summation order is fixed -> deterministic.
__device__ __forceinline__ float warp_reduce16(float (&v)[16], int lane) {
  {
    const bool hi = lane & 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float send = hi ? v[i] : v[i + 8];
      float keep = hi ? v[i + 8] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  }
  {
    const bool hi = lane & 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float send = hi ? v[i] : v[i + 4];
      float keep = hi ? v[i + 4] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
  }
  {
    const bool hi = lane & 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float send = hi ? v[i] : v[i + 2];
      float keep = hi ? v[i + 2] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
  }
  {
    const bool hi = lane & 2;
    float send = hi ? v[0] : v[1];
    float keep = hi ? v[1] : v[0];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
  return v[0];
}
__device__ __forceinline__ int warp_reduce16_slot(int lane) {
  return ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
}

// ---------------------------------------------------------------------------------------------
// Memory helpers, mbarrier + bulk asynchronous copy
// ---------------------------------------------------------------------------------------------
#if defined(PDB_EMU) && defined(__CUDACC__)
#error "PDB_EMU is the CPU test harness of tests/host/cuda_emu.h; it must never be defined in an nvcc (product) build"
#endif
#ifdef PDB_EMU
// TEST HARNESS ONLY (tests/host/cuda_emu.h): the inline-PTX helpers below restated for the CPU emulation that runs these
// kernels unmodified on the host.  Never defined in a product build (nvcc does not see PDB_EMU).
inline float4 ld_stream_f4(const float4* p) { return *p; }
inline unsigned ld_acquire_u32(const unsigned* p) {
  sched_yield();  // the poller spins on another OS thread's progress
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
}
inline unsigned ld_relaxed_u32(const unsigned* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
inline void red_release_add_u32(unsigned* p, unsigned v) { __atomic_fetch_add(p, v, __ATOMIC_RELEASE); }
inline void st_ll(unsigned long long* p, unsigned bits, unsigned tag) {
  __atomic_store_n(p, ((unsigned long long)tag << 32) | (unsigned long long)bits, __ATOMIC_RELAXED);
}
inline unsigned long long ld_ll(const unsigned long long* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
inline void pdl_wait() {}
inline void pdl_trigger() {}
inline void ld_ll2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  a = __atomic_load_n(p, __ATOMIC_RELAXED);
  b = __atomic_load_n(p + 1, __ATOMIC_RELAXED);
}
inline void st_ll2(unsigned long long* p, unsigned bits0, unsigned bits1, unsigned tag) {
  st_ll(p, bits0, tag);
  st_ll(p + 1, bits1, tag);
}
// {fp32 sum, fp32 arrivals} accumulators of the one-hop all-reduce: the pair is updated / read as ONE 64-bit unit here
inline void red_pair_add(float* p, float v) {
  unsigned long long* u = reinterpret_cast<unsigned long long*>(p);
  unsigned long long old = __atomic_load_n(u, __ATOMIC_RELAXED);
  for (;;) {
    float f[2];
    memcpy(f, &old, 8);
    f[0] += v;
    f[1] += 1.0f;
    unsigned long long want;
    memcpy(&want, f, 8);
    if (__atomic_compare_exchange_n(u, &old, want, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return;
  }
}
inline float2 ld_pair(const float* p) {
  const unsigned long long w = __atomic_load_n(reinterpret_cast<const unsigned long long*>(p), __ATOMIC_RELAXED);
  float f[2];
  memcpy(f, &w, 8);
  return make_float2(f[0], f[1]);
}
inline void st_pair_zero(float* p) { __atomic_store_n(reinterpret_cast<unsigned long long*>(p), 0ull, __ATOMIC_RELAXED); }
inline void red_add_u64(unsigned long long* p, unsigned long long v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline void fence_gpu() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void ll_backoff() {  // the poller waits for other CTAs (OS threads): let the CTA's other threads publish first
  emu::yield();
  sched_yield();
}
inline uint32_t smem_u32(const void* p) { return emu::shared_addr(p); }
inline void mbar_init(uint32_t bar, uint32_t count) { emu::mbar_init(bar, count); }
inline void mbar_fence_init() {}
inline void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) { emu::mbar_arrive_expect_tx(bar, bytes); }
inline bool mbar_try_wait(uint32_t bar, uint32_t parity) { return emu::mbar_try_wait(bar, parity); }
inline void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
inline void bulk_copy_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) { emu::bulk_copy_g2s(dst_smem, src, bytes, bar); }
inline uint64_t l2_policy_evict_first() { return 0; }
inline void bulk_copy_g2s_hint(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t) { emu::bulk_copy_g2s(dst_smem, src, bytes, bar); }
#else
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add_u32(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Flag-carrying exchange words: ONE 64-bit relaxed store publishes {32-bit payload, 32-bit tag}.  A 64-bit scalar access
// is single-copy atomic, so a reader that sees the expected tag has the payload that was stored with it -- no fence, no
// separate flag, no barrier counter (the protocol NCCL calls "LL").  Loads and stores go to L2 (gpu scope).
__device__ __forceinline__ void st_ll(unsigned long long* p, unsigned bits, unsigned tag) {
  const unsigned long long w = ((unsigned long long)tag << 32) | (unsigned long long)bits;
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ unsigned long long ld_ll(const unsigned long long* p) {
  unsigned long long w;
  asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
  return w;
}
// Programmatic dependent launch (kernels chained inside the tensor-core engine's step graph): `pdl_trigger` lets the next kernel
// of the chain start its prologue (barrier init, descriptor prefetch) while this one is still running;
// `pdl_wait` blocks until the previous kernel has completed and its writes are visible.  Both are no-ops in a kernel that was
// not launched with the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// two neighbouring words with one 16-byte access (16-byte aligned); each 64-bit element is single-copy atomic on its own
__device__ __forceinline__ void ld_ll2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.b64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_ll2(unsigned long long* p, unsigned bits0, unsigned bits1, unsigned tag) {
  const unsigned long long w0 = ((unsigned long long)tag << 32) | (unsigned long long)bits0;
  const unsigned long long w1 = ((unsigned long long)tag << 32) | (unsigned long long)bits1;
  asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1,%2};" ::"l"(p), "l"(w0), "l"(w1) : "memory");
}
__device__ __forceinline__ void ll_backoff() {}
// One-hop all-reduce accumulators: {fp32 sum, fp32 arrivals} in one 8-byte word.  ONE vector reduction adds {v, 1.0} to the
// pair (red.v2.f32, sm_90+); a reader that sees the expected number of arrivals has the complete sum.  PTX only promises
// per-element atomicity of a vector reduction; on this hardware both elements of the 8-byte-aligned pair are applied by the
// L2 reduction unit in one pass (tools/xchg_probe.cu mode 8 watches for torn pairs).
__device__ __forceinline__ void red_pair_add(float* p, float v) {
  asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v), "f"(1.0f) : "memory");
}
__device__ __forceinline__ float2 ld_pair(const float* p) {
  float2 v;
  asm volatile("ld.relaxed.gpu.global.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_pair_zero(float* p) {
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(0ull) : "memory");
}
__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void fence_gpu() { __threadfence(); }

// mbarrier + bulk asynchronous copy (global -> shared, completion counted in bytes on an mbarrier)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok)
               : "r"(bar), "r"(parity)
               : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk copy executed by the TMA unit: `bytes` (multiple of 16) from global to this CTA's shared memory
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// The same with an L2 eviction policy: the match stream of a big sequence (414 MB per inner iteration at config 5) passes
// through L2 exactly once per iteration and would otherwise evict the few hot lines every CTA polls and adds to (the exchange
// accumulators: 3.2 GB of DRAM write-backs per launch and DRAM-latency polls without the hint).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_copy_g2s_hint(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar), "l"(policy)
               : "memory");
}
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
#endif

// Sum over `count` publishers of word `e` of an exchange buffer laid out [publisher][stride] (ascending publisher order ->
// the same bits in every reader).  Polls until every word carries `tag`; up to kLlBatch loads in flight per thread.
// kInt: the payload is an int32 (exact sum) instead of an fp32.
constexpr int kLlBatch = 16;
template <bool kInt>
__device__ __forceinline__ unsigned ll_sum(const unsigned long long* base, size_t stride, int count, unsigned tag) {
  float fsum = 0.f;
  int isum = 0;
  for (int c0 = 0; c0 < count; c0 += kLlBatch) {
    unsigned long long w[kLlBatch];
    bool ok;
    do {
      ok = true;
#pragma unroll
      for (int k = 0; k < kLlBatch; ++k) {  // past the end: the last publisher again (keeps the batch branch-free, in registers)
        w[k] = ld_ll(base + (size_t)min(c0 + k, count - 1) * stride);
        ok = ok && ((unsigned)(w[k] >> 32) == tag);
      }
      if (!ok) ll_backoff();
    } while (!ok);
#pragma unroll
    for (int k = 0; k < kLlBatch; ++k) {
      const bool in = c0 + k < count;
      if (kInt) isum += in ? (int)(unsigned)w[k] : 0;
      else fsum += in ? __uint_as_float((unsigned)w[k]) : 0.f;  // + 0.f of a padding slot leaves the sum bit-identical
    }
  }
  return kInt ? (unsigned)isum : __float_as_uint(fsum);
}

// The same barrier executed by ONE warp per CTA (the rest of the CTA waits at a later __syncthreads).
// All 32 lanes may have issued global atomics before; __syncwarp orders them before lane 0's release.
__device__ __forceinline__ void warp_group_barrier(unsigned* counter, unsigned target) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) {
    red_release_add_u32(counter, 1u);
    while (ld_acquire_u32(counter) < target) {
    }
  }
  __syncwarp();
}

}  // namespace pdb
