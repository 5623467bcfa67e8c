// Microbenchmark (GPU box only): latency of one grid-wide all-reduce of a small fp32 vector between the persistent CTAs of
// a cooperative launch -- the exchange that closes every inner iteration of the GGS kernel (csrc/ggs.cuh).
//
//   mode 0  round-1 scheme: red.global.add into one 128-byte line per value, release/acquire counter barrier, read-back
//   mode 1  flag-carrying words ("LL": one 64-bit store = {fp32 value, iteration tag}), ONE level: every CTA reads all slots
//   mode 3  two levels with plain data + one release flag per slot (flag-first polling)
//   mode 4  hop calibration (two CTAs bounce one word)
//   mode 6  two levels with 16-byte {3 values, tag} words (counts torn words)
//   mode 7  mode 2 with 16 loads in flight per thread (the kernel's setting)
//   mode 8  ONE hop: red.v2.f32 {value, 1.0} into per-value accumulators, poll the arrival count (checks vector atomicity)
//   mode 9  mode 7 + nanosleep back-off;  mode 10  poll one word per slot first, then read;  mode 11  three hops, minimal traffic
//   mode 2  LL, TWO levels: groups of S CTAs, the group leader sums its group's slots and publishes a group slot,
//           every CTA then reads the G group slots
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a tools/xchg_probe.cu -o build/xchg_probe
//   build/xchg_probe [words=148] [iters=20000]
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

__device__ __forceinline__ void st_ll(unsigned long long* p, float v, unsigned tag) {
  const unsigned long long w = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
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

// sum of word e over `count` publishers [publisher][words], polling for `tag`; B loads in flight
template <int B>
__device__ __forceinline__ float ll_sum_f(const unsigned long long* base, size_t stride, int count, unsigned tag) {
  float sum = 0.f;
  for (int c0 = 0; c0 < count; c0 += B) {
    unsigned long long w[B];
    bool ok;
    do {
      ok = true;
#pragma unroll
      for (int k = 0; k < B; ++k) {
        w[k] = ld_ll(base + (size_t)min(c0 + k, count - 1) * stride);
        ok = ok && ((unsigned)(w[k] >> 32) == tag);
      }
    } while (!ok);
#pragma unroll
    for (int k = 0; k < B; ++k) sum += (c0 + k < count) ? __uint_as_float((unsigned)w[k]) : 0.f;
  }
  return sum;
}
__device__ __forceinline__ void st_v4(float4* p, float4 v) {
  asm volatile("st.relaxed.gpu.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_v4(const float4* p) {
  float4 v;
  asm volatile("ld.relaxed.gpu.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ void red_v2(float* p, float a, float b) {
  asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float2 ld_f2(const float* p) {
  float2 v;
  asm volatile("ld.relaxed.gpu.global.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}

struct Params {
  int mode, words, iters, S, G, replicas;
  float* acc;                 // mode 0: [3][words*32]
  unsigned* bar;              // mode 0
  unsigned long long* slot1;  // [2][ctas][words]
  unsigned long long* slot2;  // [2][replicas][G][words]
  unsigned* flags;            // modes 3: [2][ctas + G] flag words, one 128-byte line each
  float* plain1;              // mode 3: [2][ctas][words]
  float* plain2;              // mode 3: [2][G][words]
  float4* vec1;               // mode 6: [2][ctas][words/3+1]
  float4* vec2;               // mode 6: [2][G][words/3+1]
  unsigned* torn;             // mode 6: count of torn 16-byte words observed
  float* acc2;                // mode 8: [3][words][stride floats] {sum, arrivals}
  int stride;                 // mode 8: floats between two accumulators (8 = 32 B, 32 = 128 B)
  int backoff;                // modes 9: nanoseconds between poll retries
  float* out;                 // [ctas] checksum
  long long* cycles;          // [ctas]
};

__global__ void __launch_bounds__(512, 1) xchg_kernel(const Params P) {
  extern __shared__ float s_sum[];
  const int tid = threadIdx.x, cta = blockIdx.x, C = gridDim.x;
  float mine = 1.0f + 1e-3f * (float)(cta % 7);  // this CTA's contribution per word (changes per iteration below)
  float check = 0.f;
  const long long t0 = clock64();
  for (int it = 0; it < P.iters; ++it) {
    const unsigned tag = (unsigned)it + 1u;
    const float contrib = mine + (float)(it & 3);
    if (P.mode == 0) {
      float* acc = P.acc + (size_t)(it % 3) * P.words * 32;
      if (tid < 32)
        for (int e = tid; e < P.words; e += 32) atomicAdd(&acc[e * 32], contrib);
      if (tid < 32) {
        __syncwarp();
        if (tid == 0) {
          red_release_add_u32(P.bar, 1u);
          while (ld_acquire_u32(P.bar) < tag * (unsigned)C) {
          }
        }
        __syncwarp();
        if (cta == 0) {
          float* old = P.acc + (size_t)((it + 2) % 3) * P.words * 32;
          for (int e = tid; e < P.words; e += 32) old[e * 32] = 0.f;
        }
        for (int e = tid; e < P.words; e += 32) s_sum[e] = __ldcg(&acc[e * 32]);
      }
      __syncthreads();
    } else if (P.mode == 1) {
      unsigned long long* mys = P.slot1 + ((size_t)(it & 1) * C + cta) * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) st_ll(mys + e, contrib, tag);
      const unsigned long long* base = P.slot1 + (size_t)(it & 1) * C * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) {
        float sum = 0.f;
        for (int c0 = 0; c0 < C; c0 += 8) {
          unsigned long long w[8];
          bool ok;
          do {
            ok = true;
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (c0 + k < C) {
                w[k] = ld_ll(base + (size_t)(c0 + k) * P.words + e);
                ok &= (unsigned)(w[k] >> 32) == tag;
              }
          } while (!ok);
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (c0 + k < C) sum += __uint_as_float((unsigned)w[k]);
        }
        s_sum[e] = sum;
      }
      __syncthreads();
    } else if (P.mode == 3) {
      // flag-first: plain data stores, __syncthreads, ONE release store of a per-slot flag; readers poll the flags with one
      // lane per slot, then read the data with plain (L2) loads
      const int S = P.S, G = P.G;
      float* mys = P.plain1 + ((size_t)(it & 1) * C + cta) * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) __stcg(mys + e, contrib);
      __syncthreads();
      unsigned* fl = P.flags + (size_t)(it & 1) * (C + G) * 32;
      if (tid == 0) st_release_u32(fl + cta * 32, tag);
      const int g = cta / S;
      if (cta % S == 0) {
        const int c_lo = g * S, c_hi = min(C, c_lo + S);
        if (tid < c_hi - c_lo) while (ld_acquire_u32(fl + (c_lo + tid) * 32) != tag) {}
        __syncthreads();
        const float* base = P.plain1 + (size_t)(it & 1) * C * P.words;
        float* dst = P.plain2 + ((size_t)(it & 1) * G + g) * P.words;
        for (int e = tid; e < P.words; e += blockDim.x) {
          float sum = 0.f;
          for (int c = c_lo; c < c_hi; ++c) sum += __ldcg(base + (size_t)c * P.words + e);
          __stcg(dst + e, sum);
        }
        __syncthreads();
        if (tid == 0) st_release_u32(fl + (C + g) * 32, tag);
      }
      if (tid < G) while (ld_acquire_u32(fl + (C + tid) * 32) != tag) {}
      __syncthreads();
      const float* base2 = P.plain2 + (size_t)(it & 1) * G * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) {
        float sum = 0.f;
        for (int gg = 0; gg < G; ++gg) sum += __ldcg(base2 + (size_t)gg * P.words + e);
        s_sum[e] = sum;
      }
      __syncthreads();
    } else if (P.mode == 6) {
      // 16-byte words {v0, v1, v2, tag}: three values per store; NOT formally single-copy atomic -> torn words are counted
      const int S = P.S, G = P.G, W4 = (P.words + 2) / 3;
      float4* mys = P.vec1 + ((size_t)(it & 1) * C + cta) * W4;
      for (int e = tid; e < W4; e += blockDim.x) st_v4(mys + e, make_float4(contrib, contrib, contrib, __uint_as_float(tag)));
      const int g = cta / S;
      auto sum4 = [&](const float4* base, size_t stride, int count) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c0 = 0; c0 < count; c0 += 8) {
          float4 w[8];
          bool ok;
          do {
            ok = true;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              w[k] = ld_v4(base + (size_t)min(c0 + k, count - 1) * stride);
              ok = ok && (__float_as_uint(w[k].w) == tag);
            }
          } while (!ok);
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (c0 + k < count) {
              if (w[k].x != w[k].y || w[k].y != w[k].z) atomicAdd(P.torn, 1u);
              acc.x += w[k].x; acc.y += w[k].y; acc.z += w[k].z;
            }
        }
        return acc;
      };
      if (cta % S == 0) {
        const int c_lo = g * S, c_n = min(C, c_lo + S) - c_lo;
        const float4* base = P.vec1 + ((size_t)(it & 1) * C + c_lo) * W4;
        for (int e = tid; e < W4; e += blockDim.x) {
          float4 a = sum4(base + e, W4, c_n);
          a.y = a.x; a.z = a.x;  // keep the torn-word check meaningful at level 2
          a.w = __uint_as_float(tag);
          st_v4(P.vec2 + ((size_t)(it & 1) * G + g) * W4 + e, a);
        }
      }
      const float4* base2 = P.vec2 + (size_t)(it & 1) * G * W4;
      for (int e = tid; e < W4; e += blockDim.x) {
        const float4 a = sum4(base2 + e, W4, G);
        s_sum[3 * e] = a.x;
        if (3 * e + 1 < P.words) s_sum[3 * e + 1] = a.y;
        if (3 * e + 2 < P.words) s_sum[3 * e + 2] = a.z;
      }
      __syncthreads();
    } else if (P.mode == 8) {
      // ONE hop: every CTA adds {value, 1.0} to each accumulator with one vector reduction (red.v2.f32); everybody polls the
      // accumulators until the arrival count is complete.  Triple-buffered; CTA 0 zeroes the buffer used two iterations ago.
      // The value added is exactly 1.0 here, so a consistent {sum, arrivals} pair always has sum == arrivals: any other
      // observation means the two elements of the vector reduction were applied separately (counted in `torn`).
      float* acc = P.acc2 + (size_t)(it % 3) * P.words * P.stride;
      for (int e = tid; e < P.words; e += blockDim.x) red_v2(acc + (size_t)e * P.stride, 1.0f, 1.0f);
      for (int e = tid; e < P.words; e += blockDim.x) {
        float2 v;
        do {
          v = ld_f2(acc + (size_t)e * P.stride);
          if (v.x != v.y) atomicAdd(P.torn, 1u);
        } while (v.y != (float)C);
        s_sum[e] = v.x;
      }
      if (cta == 0) {
        float* old = P.acc2 + (size_t)((it + 2) % 3) * P.words * P.stride;
        for (int e = tid; e < P.words; e += blockDim.x) *reinterpret_cast<float2*>(old + (size_t)e * P.stride) = make_float2(0.f, 0.f);
        __threadfence();
      }
      __syncthreads();
    } else if (P.mode == 9 || P.mode == 10) {
      // mode 9: mode 7 + nanosleep between poll retries; mode 10: lanes of warp 0 first poll the LAST word of every slot
      // (one load per slot per retry), then everybody reads (and verifies) the slots once
      const int S = P.S, G = P.G;
      unsigned long long* mys = P.slot1 + ((size_t)(it & 1) * C + cta) * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) st_ll(mys + e, contrib, tag);
      const int g = cta / S;
      auto sum_slots = [&](const unsigned long long* base, int count, int e) {
        float sum = 0.f;
        unsigned long long w[16];
        bool ok;
        do {
          ok = true;
#pragma unroll
          for (int k = 0; k < 16; ++k) {
            w[k] = ld_ll(base + (size_t)min(k, count - 1) * P.words + e);
            ok = ok && ((unsigned)(w[k] >> 32) == tag);
          }
          if (!ok && P.backoff) __nanosleep(P.backoff);
        } while (!ok);
#pragma unroll
        for (int k = 0; k < 16; ++k) sum += (k < count) ? __uint_as_float((unsigned)w[k]) : 0.f;
        return sum;
      };
      auto wait_last_word = [&](const unsigned long long* base, int count) {
        if (tid < 32) {
          bool ok;
          do {
            ok = true;
            for (int k = tid; k < count; k += 32) ok = ok && ((unsigned)(ld_ll(base + (size_t)k * P.words + P.words - 1) >> 32) == tag);
            ok = __all_sync(0xffffffffu, ok);
            if (!ok && P.backoff) __nanosleep(P.backoff);
          } while (!ok);
        }
        __syncthreads();
      };
      if (cta % S == 0) {
        const int c_lo = g * S, c_n = min(C, c_lo + S) - c_lo;
        const unsigned long long* base = P.slot1 + ((size_t)(it & 1) * C + c_lo) * P.words;
        if (P.mode == 10) wait_last_word(base, c_n);
        for (int e = tid; e < P.words; e += blockDim.x)
          st_ll(P.slot2 + ((size_t)(it & 1) * G + g) * P.words + e, sum_slots(base, c_n, e), tag);
      }
      const unsigned long long* base2 = P.slot2 + (size_t)(it & 1) * G * P.words;
      if (P.mode == 10) wait_last_word(base2, G);
      for (int e = tid; e < P.words; e += blockDim.x) s_sum[e] = sum_slots(base2, G, e);
      __syncthreads();
    } else if (P.mode == 11) {
      // THREE hops, minimal traffic: members -> group leader -> all leaders sum the G group slots -> each leader publishes the
      // total in its group's result slot -> members read ONE slot (12 readers per slot instead of 148 readers per group slot)
      const int S = P.S, G = P.G;
      unsigned long long* mys = P.slot1 + ((size_t)(it & 1) * C + cta) * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) st_ll(mys + e, contrib, tag);
      const int g = cta / S;
      unsigned long long* result = P.slot2 + ((size_t)(2 + (it & 1)) * G + g) * P.words;  // second half of slot2: result slots
      if (cta % S == 0) {
        const int c_lo = g * S, c_n = min(C, c_lo + S) - c_lo;
        const unsigned long long* base = P.slot1 + ((size_t)(it & 1) * C + c_lo) * P.words;
        for (int e = tid; e < P.words; e += blockDim.x)
          st_ll(P.slot2 + ((size_t)(it & 1) * G + g) * P.words + e, ll_sum_f<16>(base + e, P.words, c_n, tag), tag);
        const unsigned long long* base2 = P.slot2 + (size_t)(it & 1) * G * P.words;
        for (int e = tid; e < P.words; e += blockDim.x) {
          const float total = ll_sum_f<16>(base2 + e, P.words, G, tag);
          st_ll(result + e, total, tag);
          s_sum[e] = total;
        }
      } else {
        for (int e = tid; e < P.words; e += blockDim.x) s_sum[e] = ll_sum_f<16>(result + e, P.words, 1, tag);
      }
      __syncthreads();
    } else if (P.mode == 7) {
      // mode 2 with 16 loads in flight per thread (what csrc/ggs.cuh does)
      const int S = P.S, G = P.G;
      unsigned long long* mys = P.slot1 + ((size_t)(it & 1) * C + cta) * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) st_ll(mys + e, contrib, tag);
      const int g = cta / S;
      if (cta % S == 0) {
        const int c_lo = g * S, c_n = min(C, c_lo + S) - c_lo;
        const unsigned long long* base = P.slot1 + ((size_t)(it & 1) * C + c_lo) * P.words;
        for (int e = tid; e < P.words; e += blockDim.x)
          st_ll(P.slot2 + ((size_t)(it & 1) * G + g) * P.words + e, ll_sum_f<16>(base + e, P.words, c_n, tag), tag);
      }
      const unsigned long long* base2 = P.slot2 + (size_t)(it & 1) * G * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) s_sum[e] = ll_sum_f<16>(base2 + e, P.words, G, tag);
      __syncthreads();
    } else if (P.mode == 4) {
      // hop calibration: CTA 0 and CTA 1 bounce one word; everybody else idles (two hops per iteration)
      if (cta < 2 && tid == 0) {
        unsigned long long* a = P.slot1, *b = P.slot1 + 64;
        if (cta == 0) {
          st_ll(a, 1.0f, tag);
          while ((unsigned)(ld_ll(b) >> 32) != tag) {}
        } else {
          while ((unsigned)(ld_ll(a) >> 32) != tag) {}
          st_ll(b, 1.0f, tag);
        }
      }
      if (tid < P.words + 1) s_sum[tid] = 0.f;
      __syncthreads();
    } else {
      const int S = P.S, G = P.G;
      unsigned long long* mys = P.slot1 + ((size_t)(it & 1) * C + cta) * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) st_ll(mys + e, contrib, tag);
      const int g = cta / S;
      if (cta % S == 0) {  // group leader: sum the group's slots, publish
        const int c_lo = g * S, c_hi = min(C, c_lo + S);
        const unsigned long long* base = P.slot1 + (size_t)(it & 1) * C * P.words;
        for (int e = tid; e < P.words; e += blockDim.x) {
          float sum = 0.f;
          for (int c0 = c_lo; c0 < c_hi; c0 += 8) {
            unsigned long long w[8];
            bool ok;
            do {
              ok = true;
#pragma unroll
              for (int k = 0; k < 8; ++k)
                if (c0 + k < c_hi) {
                  w[k] = ld_ll(base + (size_t)(c0 + k) * P.words + e);
                  ok &= (unsigned)(w[k] >> 32) == tag;
                }
            } while (!ok);
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (c0 + k < c_hi) sum += __uint_as_float((unsigned)w[k]);
          }
          for (int r = 0; r < P.replicas; ++r)
            st_ll(P.slot2 + (((size_t)(it & 1) * P.replicas + r) * G + g) * P.words + e, sum, tag);
        }
      }
      const unsigned long long* base2 = P.slot2 + ((size_t)(it & 1) * P.replicas + (cta % P.replicas)) * G * P.words;
      for (int e = tid; e < P.words; e += blockDim.x) {
        float sum = 0.f;
        for (int g0 = 0; g0 < G; g0 += 8) {
          unsigned long long w[8];
          bool ok;
          do {
            ok = true;
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (g0 + k < G) {
                w[k] = ld_ll(base2 + (size_t)(g0 + k) * P.words + e);
                ok &= (unsigned)(w[k] >> 32) == tag;
              }
          } while (!ok);
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (g0 + k < G) sum += __uint_as_float((unsigned)w[k]);
        }
        s_sum[e] = sum;
      }
      __syncthreads();
    }
    if (tid == 0) {
      check += s_sum[0] + s_sum[P.words - 1];
      mine += 1e-6f * s_sum[0];  // the next contribution depends on this result (no overlap across iterations)
    }
    mine = __shfl_sync(0xffffffffu, mine, 0);
    __syncthreads();
    if (tid >= 32) mine = 0.f;  // only warp 0's value is used; keep the dependency simple
    if (tid == 0) s_sum[P.words] = mine;
    __syncthreads();
    mine = s_sum[P.words];
    __syncthreads();
  }
  if (tid == 0) {
    P.out[cta] = check;
    P.cycles[cta] = clock64() - t0;
  }
}

int main(int argc, char** argv) {
  const int words = argc > 1 ? atoi(argv[1]) : 148;
  const int iters = argc > 2 ? atoi(argv[2]) : 20000;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("device %s, %d SMs, clock %d kHz\n", prop.name, sms, prop.clockRate);
  // (a) how many CTAs of the GGS shape (512 threads, ~200 KB dynamic shared memory) can be co-resident as clusters?
  for (int cs : {1, 2, 4, 8, 16}) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(sms / cs * cs);
    cfg.blockDim = dim3(512);
    cfg.dynamicSmemBytes = 200 * 1024;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaFuncSetAttribute(xchg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (cs > 8) cudaFuncSetAttribute(xchg_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    int n = 0;
    cudaError_t e = cudaOccupancyMaxActiveClusters(&n, xchg_kernel, &cfg);
    printf("cluster size %2d: max active clusters %d (%d CTAs) %s\n", cs, n, n * cs, e == cudaSuccess ? "" : cudaGetErrorString(e));
  }
  cudaGetLastError();
  Params P = {};
  P.words = words;
  P.iters = iters;
  const int maxC = sms;
  CK(cudaMalloc(&P.acc, sizeof(float) * 3 * words * 32));
  CK(cudaMalloc(&P.bar, 256));
  CK(cudaMalloc(&P.slot1, sizeof(unsigned long long) * 2 * maxC * words));
  CK(cudaMalloc(&P.slot2, sizeof(unsigned long long) * 2 * 8 * 64 * words));
  CK(cudaMalloc(&P.flags, sizeof(unsigned) * 2 * (maxC + 64) * 32));
  CK(cudaMalloc(&P.plain1, sizeof(float) * 2 * maxC * words));
  CK(cudaMalloc(&P.plain2, sizeof(float) * 2 * 64 * words));
  CK(cudaMalloc(&P.vec1, sizeof(float4) * 2 * maxC * (words / 3 + 1)));
  CK(cudaMalloc(&P.vec2, sizeof(float4) * 2 * 64 * (words / 3 + 1)));
  CK(cudaMalloc(&P.torn, 256));
  CK(cudaMalloc(&P.acc2, sizeof(float) * 3 * words * 32));
  CK(cudaMemset(P.torn, 0, 256));
  CK(cudaMalloc(&P.out, sizeof(float) * maxC));
  CK(cudaMalloc(&P.cycles, sizeof(long long) * maxC));
  CK(cudaFuncSetAttribute(xchg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  struct Case { int mode, C, S, rep; };
  std::vector<Case> cases;
  // {mode, ctas, S, rep}; for mode 8 S = accumulator stride in floats; for mode 9/10 rep = nanosleep ns
  for (int C : {18, 74, 148}) {
    cases.push_back({0, C, 0, 1});
    cases.push_back({8, C, 8, 1});
    cases.push_back({8, C, 32, 1});
    for (int S : {10, 12}) {
      if (S >= C) continue;
      cases.push_back({7, C, S, 1});
      cases.push_back({9, C, S, 100});
      cases.push_back({9, C, S, 400});
      cases.push_back({10, C, S, 0});
      cases.push_back({10, C, S, 100});
      cases.push_back({11, C, S, 1});
    }
  }
  for (const Case& c : cases) {
    P.mode = c.mode;
    P.S = c.S;
    P.G = c.S ? (c.C + c.S - 1) / c.S : 0;
    P.replicas = 1;
    P.stride = c.S;
    P.backoff = c.rep;
    CK(cudaMemset(P.torn, 0, 256));
    CK(cudaMemset(P.acc, 0, sizeof(float) * 3 * words * 32));
    CK(cudaMemset(P.bar, 0, 256));
    CK(cudaMemset(P.slot1, 0, sizeof(unsigned long long) * 2 * maxC * words));
    CK(cudaMemset(P.slot2, 0, sizeof(unsigned long long) * 2 * 8 * 64 * words));
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    void* args[] = {&P};
    float best = 1e30f;
    float chk = 0.f;
    for (int rep = 0; rep < 3; ++rep) {
      CK(cudaMemset(P.bar, 0, 256));
      CK(cudaMemset(P.acc, 0, sizeof(float) * 3 * words * 32));
      CK(cudaMemset(P.slot1, 0, sizeof(unsigned long long) * 2 * maxC * words));
      CK(cudaMemset(P.slot2, 0, sizeof(unsigned long long) * 2 * 8 * 64 * words));
      CK(cudaMemset(P.flags, 0, sizeof(unsigned) * 2 * (maxC + 64) * 32));
      CK(cudaMemset(P.vec1, 0, sizeof(float4) * 2 * maxC * (words / 3 + 1)));
      CK(cudaMemset(P.vec2, 0, sizeof(float4) * 2 * 64 * (words / 3 + 1)));
      CK(cudaMemset(P.acc2, 0, sizeof(float) * 3 * words * 32));
      CK(cudaEventRecord(a));
      CK(cudaLaunchCooperativeKernel((void*)xchg_kernel, dim3(c.C), dim3(512), args, 64 * 1024, 0));
      CK(cudaEventRecord(b));
      CK(cudaEventSynchronize(b));
      float ms;
      CK(cudaEventElapsedTime(&ms, a, b));
      if (ms < best) best = ms;
      CK(cudaMemcpy(&chk, P.out, sizeof(float), cudaMemcpyDeviceToHost));
    }
    unsigned torn = 0;
    CK(cudaMemcpy(&torn, P.torn, 4, cudaMemcpyDeviceToHost));
    printf("mode %d  ctas %3d  S %2d G %2d rep %d : %8.3f us per all-reduce   (check %.3f, torn %u)\n", c.mode, c.C, c.S, P.G, c.rep,
           best * 1e3f / iters, chk, torn);
  }
  return 0;
}
