// C-ABI entry points: context, correspondences, Sampson evaluation, geometry-guided sampling.
// (include/posediff_b200.h documents which reference call site each one replaces.)
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <new>
#include <thread>

#include "context.cuh"
#include "ggs.cuh"

using namespace pdb;

namespace {
std::string g_create_error;

constexpr int kGgsBatchMax = 16;
struct GgsBatch {
  GgsProblem prob[kGgsBatchMax];
};

template <bool kEval, bool kPaired, bool kProbe = false, bool kLean = false>
__global__ void __launch_bounds__(kGgsThreads, 1)
ggs_entry(const __grid_constant__ GgsBatch batch, const __grid_constant__ GgsParams P);

// Exchange workspace of one sequence: double-buffered slots of its CTAs (xch1) and of its group leaders (xch2).
size_t ggs_ws_slots_bytes(int frames, int cpp, int group) {
  const size_t words = 2 * (size_t)(cpp + ggs_xch_groups(cpp, group)) * ggs_xch_words(frames);
  return (words * sizeof(unsigned long long) + 255) / 256 * 256;
}
size_t ggs_ws_per_problem(int frames, int cpp, int group) {  // slots + the three accumulator buffers of the one-hop exchange
  return ggs_ws_slots_bytes(frames, cpp, group) + (sizeof(float) * 3 * (size_t)ggs_xch_words(frames) * kAccStride + 255) / 256 * 256;
}

int env_int(const char* name, int fallback) {
  const char* v = getenv(name);
  return (v && v[0]) ? atoi(v) : fallback;
}

// CTAs per sequence of one launch of `nprob` sequences (one CTA per SM, at least ~1 round per warp) and the exchange
// group size.  PDB_GGS_CPP / PDB_GGS_GROUP are tuning overrides (an upper bound on the CTAs per sequence / the group size).
void ggs_plan(const Context* ctx, int nprob, long long max_rounds, int* cpp_out, int* group_out) {
  int cpp = ctx->sm_count / nprob;
  if (cpp < 1) cpp = 1;
  long long want = max_rounds / 32;
  if (want < 1) want = 1;
  if (cpp > want) cpp = (int)want;
  const int cap = env_int("PDB_GGS_CPP", 0);
  if (cap >= 1 && cpp > cap) cpp = cap;
  int group = env_int("PDB_GGS_GROUP", kXchGroupDefault);
  if (group < 2) group = 2;
  if (cpp <= 2 * group) group = cpp;  // few CTAs: one level (every CTA sums every slot)
  *cpp_out = cpp;
  *group_out = group;
}
int ggs_xch_mode() { return env_int("PDB_GGS_XCH", 1) == 0 ? 0 : 1; }  // PDB_GGS_XCH=0: exchange through flag-carrying slots
}  // namespace

extern "C" {

int pdb_abi_version(void) { return PDB_ABI_VERSION; }

const char* pdb_last_error(const pdb_context* ctx) {
  if (!ctx) return g_create_error.c_str();
  return reinterpret_cast<const Context*>(ctx)->error.c_str();
}

int pdb_create(pdb_context** out, int device_ordinal) {
  if (!out) return PDB_ERR_INVALID;
  *out = nullptr;
  int count = 0;
  cudaError_t err = cudaGetDeviceCount(&count);
  if (err != cudaSuccess || count == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(err) + " (this library has no CPU fallback)";
    return PDB_ERR_CUDA;
  }
  if (device_ordinal < 0 || device_ordinal >= count) {
    g_create_error = "device ordinal out of range";
    return PDB_ERR_INVALID;
  }
  cudaDeviceProp prop;
  if ((err = cudaGetDeviceProperties(&prop, device_ordinal)) != cudaSuccess) {
    g_create_error = cudaGetErrorString(err);
    return PDB_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    g_create_error = "posediff_b200 is built for sm_90a only; device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor);
    return PDB_ERR_CUDA;
  }
  if ((err = cudaSetDevice(device_ordinal)) != cudaSuccess) {
    g_create_error = cudaGetErrorString(err);
    return PDB_ERR_CUDA;
  }
  Context* ctx = new (std::nothrow) Context();
  if (!ctx) return PDB_ERR_CUDA;
  ctx->device = device_ordinal;
  ctx->attr = kernel_attrs(device_ordinal, count);
  ctx->sm_count = prop.multiProcessorCount;
  ctx->cc_major = prop.major;
  ctx->cc_minor = prop.minor;
  ctx->smem_optin = prop.sharedMemPerBlockOptin;
  if (const char* lay = getenv("PDB_GGS_LAYOUT")) ctx->ggs_layout = (lay[0] == 'p' && lay[1] == 'a') ? kLayoutPaired : kLayoutPlain;
  if (const char* f = getenv("PDB_DEN_FLAG")) ctx->den_flag = atoi(f) != 0;
  if (const char* f = getenv("PDB_TC_PDL")) ctx->tc_pdl = atoi(f) != 0;
  *out = reinterpret_cast<pdb_context*>(ctx);
  return PDB_OK;
}

int pdb_device_info(const pdb_context* c, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor) {
  if (!c) return PDB_ERR_INVALID;
  const Context* ctx = reinterpret_cast<const Context*>(c);
  if (sm_count) *sm_count = ctx->sm_count;
  if (cc_major) *cc_major = ctx->cc_major;
  if (cc_minor) *cc_minor = ctx->cc_minor;
  return PDB_OK;
}

int pdb_profile_enable(pdb_context* c, int32_t on) {
  if (!c) return PDB_ERR_INVALID;
  reinterpret_cast<Context*>(c)->profiling = on != 0;
  return PDB_OK;
}

int pdb_profile_read(pdb_context* c, double* ggs_ms, int64_t* ggs_launches, double* den_ms, int64_t* den_launches) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  double ms[2] = {0.0, 0.0};
  int64_t n[2] = {0, 0};
  for (auto& t : ctx->timed) {
    PDB_CUDA(ctx, cudaEventSynchronize(t.b));
    float dt = 0.f;
    PDB_CUDA(ctx, cudaEventElapsedTime(&dt, t.a, t.b));
    ms[t.kind] += dt;
    n[t.kind] += 1;
    cudaEventDestroy(t.a);
    cudaEventDestroy(t.b);
  }
  ctx->timed.clear();
  if (ggs_ms) *ggs_ms = ms[0];
  if (ggs_launches) *ggs_launches = n[0];
  if (den_ms) *den_ms = ms[1];
  if (den_launches) *den_launches = n[1];
  return PDB_OK;
}

// Debug probe: per-CTA cycle sums of the GGS stages {stage3 norms, stage1, stage2b, exchange, stage2a, iterations, next stage 0, stage3 update} (enable = 1) or of
// the fp32 denoiser kernel {barrier, tile load + LayerNorm, linear item, attention, tail, steps} (enable = 2).
int pdb_debug_ggs_clocks(pdb_context* c, int32_t enable, int64_t* out, int32_t max_ctas) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  ctx->den_clock = enable == 2;
  if (enable && !ctx->ggs_clock) {
    ctx->ggs_clock_ctas = ctx->sm_count;
    PDB_CUDA(ctx, cudaMalloc(&ctx->ggs_clock, sizeof(long long) * 8 * ctx->ggs_clock_ctas));
    PDB_CUDA(ctx, cudaMemset(ctx->ggs_clock, 0, sizeof(long long) * 8 * ctx->ggs_clock_ctas));
  }
  if (out && ctx->ggs_clock) {
    PDB_CUDA(ctx, cudaDeviceSynchronize());
    const int n = max_ctas < ctx->ggs_clock_ctas ? max_ctas : ctx->ggs_clock_ctas;
    PDB_CUDA(ctx, cudaMemcpy(out, ctx->ggs_clock, sizeof(long long) * 8 * n, cudaMemcpyDeviceToHost));
    PDB_CUDA(ctx, cudaMemset(ctx->ggs_clock, 0, sizeof(long long) * 8 * ctx->ggs_clock_ctas));
  }
  if (!enable && ctx->ggs_clock) {
    cudaFree(ctx->ggs_clock);
    ctx->ggs_clock = nullptr;
  }
  return PDB_OK;
}

int64_t pdb_launch_count(const pdb_context* c) { return c ? reinterpret_cast<const Context*>(c)->launches : 0; }

}  // extern "C"

namespace {
// Common tail of the packers: `segs` (without sentinel) are laid out in rounds, `row(src)` yields the fp32 quad of the
// src-th match in segment order.  Fills pinned staging memory (threaded for big inputs), uploads, returns the handle.
// Rows of segments [s0, s1) into the host image of the stream, in the given layout (ggs_layout.cuh); `first[s]` = index of
// the segment's first match in segment order.
template <typename Row>
void fill_segments(const std::vector<int4>& segs, const std::vector<int64_t>& first, int s0, int s1, bool paired, float4* hpts, Row row) {
  for (int s = s0; s < s1; ++s) {
    const int64_t src0 = first[s];
    const int cnt = segs[s].y;
    if (!paired) {
      float4* dst = hpts + (size_t)segs[s].x * 32;
      const int padded = (cnt + 31) / 32 * 32;
      for (int k = 0; k < cnt; ++k) dst[k] = row(src0 + k);
      for (int k = cnt; k < padded; ++k) dst[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      float* flat = reinterpret_cast<float*>(hpts);
      const long long seg_rounds = layout_seg_rounds(cnt, true);
      memset(hpts + (size_t)segs[s].x * 32, 0, sizeof(float4) * 32 * (size_t)seg_rounds);  // padding rows are zero
      for (int k = 0; k < cnt; ++k) {
        const float4 v = row(src0 + k);
        flat[layout_float_index(segs[s].x, k, 0, true)] = v.x;
        flat[layout_float_index(segs[s].x, k, 1, true)] = v.y;
        flat[layout_float_index(segs[s].x, k, 2, true)] = v.z;
        flat[layout_float_index(segs[s].x, k, 3, true)] = v.w;
      }
    }
  }
}

// Pass 1 of pdb_matches_pack: maximal runs of equal (a, b) -> segments {first_round, count, a, b}; pair index a*N+b as the
// reference (:26) computes it.  Returns the index of the first bad row, or -1.
int64_t build_segments(const int64_t* i12, int64_t m_total, int frames, bool paired, std::vector<int4>& segs, long long* rounds_out) {
  long long rounds = 0;
  for (int64_t i = 0; i < m_total;) {
    const int64_t a = i12[2 * i], b = i12[2 * i + 1];
    if (a < 0 || a >= frames || b < 0 || b >= frames) return i;
    int64_t j = i + 1;
    while (j < m_total && i12[2 * j] == a && i12[2 * j + 1] == b) ++j;
    int64_t remaining = j - i;
    while (remaining > 0) {  // keep per-segment counts inside int32
      const int64_t take = remaining > (1 << 30) ? (1 << 30) : remaining;
      segs.push_back(make_int4((int)rounds, (int)take, (int)a, (int)b));
      rounds += layout_seg_rounds(take, paired);
      remaining -= take;
    }
    i = j;
  }
  *rounds_out = rounds;
  return -1;
}

template <typename Row>
int finish_pack(Context* ctx, std::vector<int4>& segs, long long rounds, int64_t m_total, int frames, int height, int width,
                cudaStream_t st, pdb_matches** out, Row row) {
  if (rounds > 0x7fffffffLL / 32) return ctx->fail(PDB_ERR_LIMIT, "too many matches");
  const int nseg = (int)segs.size();
  const bool paired = ctx->ggs_layout == kLayoutPaired;  // the callers sized the segments with the same flag
  segs.push_back(make_int4((int)rounds, 0, 0, 0));
  const size_t pts_bytes = sizeof(float4) * ((size_t)rounds * 32 ? (size_t)rounds * 32 : 1);
  const size_t segs_bytes = sizeof(int4) * segs.size();
  const size_t stage_need = pts_bytes + segs_bytes;
  if (ctx->pin_bytes < stage_need) {
    if (ctx->pin) cudaFreeHost(ctx->pin);
    ctx->pin = nullptr;
    ctx->pin_bytes = 0;
    PDB_CUDA(ctx, cudaHostAlloc(&ctx->pin, stage_need + stage_need / 4, cudaHostAllocDefault));
    ctx->pin_bytes = stage_need + stage_need / 4;
  }
  float4* hpts = static_cast<float4*>(ctx->pin);
  int4* hsegs = reinterpret_cast<int4*>(static_cast<char*>(ctx->pin) + pts_bytes);
  memcpy(hsegs, segs.data(), segs_bytes);
  {
    std::vector<int64_t> first(nseg + 1, 0);  // first match of each segment
    for (int s = 0; s < nseg; ++s) first[s + 1] = first[s] + segs[s].y;
    auto fill = [&](int s0, int s1) { fill_segments(segs, first, s0, s1, paired, hpts, row); };
    unsigned hw = std::thread::hardware_concurrency();
    int nthreads = m_total > 200000 ? (int)(hw < 8 ? (hw ? hw : 1) : 8) : 1;
    if (nthreads > nseg) nthreads = nseg > 0 ? nseg : 1;
    if (nthreads <= 1) {
      fill(0, nseg);
    } else {  // segments split into contiguous blocks of roughly equal match counts
      std::vector<std::thread> pool;
      int s0 = 0;
      for (int t = 0; t < nthreads; ++t) {
        const int64_t target = m_total * (t + 1) / nthreads;
        int s1 = s0;
        while (s1 < nseg && first[s1 + 1] <= target) ++s1;
        if (t == nthreads - 1) s1 = nseg;
        pool.emplace_back(fill, s0, s1);
        s0 = s1;
      }
      for (auto& th : pool) th.join();
    }
  }
  Matches* m = new (std::nothrow) Matches();
  if (!m) return ctx->fail(PDB_ERR_CUDA, "out of host memory");
  m->ctx = ctx;
  m->nseg = nseg;
  m->rounds = (int)rounds;
  m->layout = paired ? kLayoutPaired : kLayoutPlain;
  m->m_total = m_total;
  m->frames = frames;
  m->height = height;
  m->width = width;
  void* dpts = nullptr;
  void* dsegs = nullptr;
  if (pool_take(ctx, &dpts, &m->pts_bytes, pts_bytes) != PDB_OK || pool_take(ctx, &dsegs, &m->segs_bytes, segs_bytes) != PDB_OK) {
    pool_give(ctx, dpts, m->pts_bytes);
    delete m;
    return PDB_ERR_CUDA;
  }
  m->pts = static_cast<float4*>(dpts);
  m->segs = static_cast<int4*>(dsegs);
  m->host_segs = segs;
  cudaError_t err = cudaMemcpyAsync(m->pts, hpts, pts_bytes, cudaMemcpyHostToDevice, st);
  if (err == cudaSuccess) err = cudaMemcpyAsync(m->segs, hsegs, segs_bytes, cudaMemcpyHostToDevice, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);  // the staging buffer is reused by the next call
  if (err != cudaSuccess) {
    pdb_matches_free(reinterpret_cast<pdb_matches*>(m));
    return ctx->fail(PDB_ERR_CUDA, "match upload failed: %s", cudaGetErrorString(err));
  }
  *out = reinterpret_cast<pdb_matches*>(m);
  return PDB_OK;
}
}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------------
// correspondences
// ------------------------------------------------------------------------------------------------
int pdb_matches_pack(pdb_context* c, const double* kp1, const double* kp2, const int64_t* i12, int64_t m_total,
                     int32_t frames, int32_t height, int32_t width, int32_t on_device, void* stream,
                     pdb_matches** out) {
  if (!c || !out) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  *out = nullptr;
  if (m_total < 0 || frames < 1 || height < 1 || width < 1) return ctx->fail(PDB_ERR_INVALID, "bad match set shape");
  if (frames > PDB_MAX_FRAMES) return ctx->fail(PDB_ERR_LIMIT, "frames %d > PDB_MAX_FRAMES %d", frames, PDB_MAX_FRAMES);
  if (m_total > 0 && (!kp1 || !kp2 || !i12)) return ctx->fail(PDB_ERR_INVALID, "null match arrays");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));

  std::vector<double> h1, h2;
  std::vector<int64_t> hi;
  if (on_device && m_total > 0) {  // bring reference-format device arrays to the host packer
    h1.resize(2 * m_total);
    h2.resize(2 * m_total);
    hi.resize(2 * m_total);
    PDB_CUDA(ctx, cudaMemcpyAsync(h1.data(), kp1, sizeof(double) * 2 * m_total, cudaMemcpyDeviceToHost, st));
    PDB_CUDA(ctx, cudaMemcpyAsync(h2.data(), kp2, sizeof(double) * 2 * m_total, cudaMemcpyDeviceToHost, st));
    PDB_CUDA(ctx, cudaMemcpyAsync(hi.data(), i12, sizeof(int64_t) * 2 * m_total, cudaMemcpyDeviceToHost, st));
    PDB_CUDA(ctx, cudaStreamSynchronize(st));
    kp1 = h1.data();
    kp2 = h2.data();
    i12 = hi.data();
  }
  std::vector<int4> segs;
  long long rounds = 0;
  const int64_t bad = build_segments(i12, m_total, frames, ctx->ggs_layout == kLayoutPaired, segs, &rounds);
  if (bad >= 0)
    return ctx->fail(PDB_ERR_INVALID, "i12[%lld] = (%lld, %lld) outside [0, %d)", (long long)bad, (long long)i12[2 * bad],
                     (long long)i12[2 * bad + 1], frames);
  return finish_pack(ctx, segs, rounds, m_total, frames, height, width, st, out, [&](int64_t src) {
    return make_float4((float)kp1[2 * src], (float)kp1[2 * src + 1], (float)kp2[2 * src], (float)kp2[2 * src + 1]);
  });
}

// Match ingestion straight from the COLMAP / hloc tables (util/match_extraction.py:50-77, colmap_keypoint_to_pytorch3d):
// keypoints per image in COLMAP pixel coordinates, raw match index pairs per image pair, crop boxes and resize scales of
// load_and_preprocess_images.  The remap  kp' = (kp - 0.5 - bbox_xy[img]) * scale[img]  is applied in float64 (numpy's
// promotion in the reference) while the rows are gathered, so the 48 B/match kp1 / kp2 / i12 arrays never exist.
int pdb_matches_pack_colmap(pdb_context* c, int32_t n_images, const void* const* keypoints, const int32_t* kp_counts,
                            int32_t kp_is_f64, int32_t n_pairs, const int32_t* pair_ids, const int32_t* const* pair_matches,
                            const int32_t* match_counts, const double* bboxes_xyxy, const double* scales, int32_t frames,
                            int32_t height, int32_t width, void* stream, pdb_matches** out) {
  if (!c || !out) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  *out = nullptr;
  if (n_images < 1 || n_pairs < 0 || frames < 1 || !keypoints || !kp_counts || !bboxes_xyxy || !scales ||
      (n_pairs > 0 && (!pair_ids || !pair_matches || !match_counts)))
    return ctx->fail(PDB_ERR_INVALID, "bad COLMAP match tables");
  if (frames > PDB_MAX_FRAMES) return ctx->fail(PDB_ERR_LIMIT, "frames %d > PDB_MAX_FRAMES %d", frames, PDB_MAX_FRAMES);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<int4> segs;
  std::vector<int> seg_pair;  // pair table row of each segment
  long long rounds = 0;
  int64_t m_total = 0;
  for (int p = 0; p < n_pairs; ++p) {
    const int r = pair_ids[2 * p], q = pair_ids[2 * p + 1];  // 1-based COLMAP image ids
    if (r < 1 || r > n_images || q < 1 || q > n_images || r - 1 >= frames || q - 1 >= frames)
      return ctx->fail(PDB_ERR_INVALID, "pair %d = (%d, %d) outside the image list", p, r, q);
    const int cnt = match_counts[p];
    if (cnt <= 0 || !pair_matches[p]) continue;  // "if pair_match is not None" (:65)
    for (int k = 0; k < cnt; ++k) {
      const int i1 = pair_matches[p][2 * k], i2 = pair_matches[p][2 * k + 1];
      if (i1 < 0 || i1 >= kp_counts[r - 1] || i2 < 0 || i2 >= kp_counts[q - 1])
        return ctx->fail(PDB_ERR_INVALID, "match %d of pair %d indexes a missing keypoint", k, p);
    }
    segs.push_back(make_int4((int)rounds, cnt, r - 1, q - 1));  // i12 = (colmap_id - 1) (:69)
    seg_pair.push_back(p);
    rounds += layout_seg_rounds(cnt, ctx->ggs_layout == kLayoutPaired);
    m_total += cnt;
  }
  std::vector<int64_t> first(segs.size() + 1, 0);
  for (size_t s2 = 0; s2 < segs.size(); ++s2) first[s2 + 1] = first[s2] + segs[s2].y;
  auto kp = [&](int img, int idx, int comp) -> double {
    const double v = kp_is_f64 ? static_cast<const double*>(keypoints[img])[2 * idx + comp]
                               : (double)(static_cast<const float*>(keypoints[img])[2 * idx + comp] - 0.5f) + 0.5;
    // float32 tables: the reference subtracts 0.5 in float32 first (numpy keeps the array dtype), then promotes
    return (v - 0.5 - bboxes_xyxy[4 * img + comp]) * scales[img];
  };
  return finish_pack(ctx, segs, rounds, m_total, frames, height, width, st, out, [&](int64_t src) {
    const int s2 = (int)(std::upper_bound(first.begin(), first.end(), src) - first.begin()) - 1;
    const int p = seg_pair[s2], k = (int)(src - first[s2]);
    const int a = segs[s2].z, b = segs[s2].w;
    const int i1 = pair_matches[p][2 * k], i2 = pair_matches[p][2 * k + 1];
    return make_float4((float)kp(a, i1, 0), (float)kp(a, i1, 1), (float)kp(b, i2, 0), (float)kp(b, i2, 1));
  });
}

void pdb_matches_free(pdb_matches* pm) {
  if (!pm) return;
  Matches* m = reinterpret_cast<Matches*>(pm);
  pool_give(m->ctx, m->pts, m->pts_bytes);  // back to the context's pool (cudaFree is slow and synchronising)
  pool_give(m->ctx, m->segs, m->segs_bytes);
  delete m;
}

int pdb_matches_info(const pdb_matches* pm, int64_t* m_total, int32_t* segments, int64_t* rounds, int32_t* frames) {
  if (!pm) return PDB_ERR_INVALID;
  const Matches* m = reinterpret_cast<const Matches*>(pm);
  if (m_total) *m_total = m->m_total;
  if (segments) *segments = m->nseg;
  if (rounds) *rounds = m->rounds;
  if (frames) *frames = m->frames;
  return PDB_OK;
}

int pdb_ggs_layout(pdb_context* c, int32_t layout) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (layout != kLayoutPlain && layout != kLayoutPaired) return ctx->fail(PDB_ERR_INVALID, "unknown stream layout %d", layout);
  ctx->ggs_layout = layout;  // applies to match sets packed from now on; existing ones keep theirs
  return PDB_OK;
}

int pdb_ggs_layout_get(const pdb_context* c) { return c ? reinterpret_cast<const Context*>(c)->ggs_layout : -1; }

// Host-only probe of the stream layout (no GPU, no context): lays reference-format matches out exactly as pdb_matches_pack
// would place them in HBM.  The CPU tests walk this image with the kernel's own partition functions (ggs_layout.cuh).
int pdb_debug_pack_layout(const double* kp1, const double* kp2, const int64_t* i12, int64_t m_total, int32_t frames, int32_t layout,
                          int32_t* segs_out, int32_t max_segs, float* pts_out, int64_t max_rounds, int32_t* nseg_out,
                          int64_t* rounds_out) {
  if (m_total < 0 || frames < 1 || (layout != kLayoutPlain && layout != kLayoutPaired) || !nseg_out || !rounds_out)
    return PDB_ERR_INVALID;
  if (m_total > 0 && (!kp1 || !kp2 || !i12)) return PDB_ERR_INVALID;
  const bool paired = layout == kLayoutPaired;
  std::vector<int4> segs;
  long long rounds = 0;
  if (build_segments(i12, m_total, frames, paired, segs, &rounds) >= 0) return PDB_ERR_INVALID;
  *nseg_out = (int32_t)segs.size();
  *rounds_out = rounds;
  if (!segs_out || !pts_out) return PDB_OK;  // size query
  if ((int64_t)segs.size() > max_segs || rounds > max_rounds) return PDB_ERR_LIMIT;
  std::vector<int64_t> first(segs.size() + 1, 0);
  for (size_t i = 0; i < segs.size(); ++i) first[i + 1] = first[i] + segs[i].y;
  fill_segments(segs, first, 0, (int)segs.size(), paired, reinterpret_cast<float4*>(pts_out), [&](int64_t src) {
    return make_float4((float)kp1[2 * src], (float)kp1[2 * src + 1], (float)kp2[2 * src], (float)kp2[2 * src + 1]);
  });
  memcpy(segs_out, segs.data(), sizeof(int4) * segs.size());
  return PDB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// GGS launch plumbing (shared with the sampler in api_sampler.cu)
// ------------------------------------------------------------------------------------------------
namespace {
template <bool kEval, bool kPaired, bool kProbe, bool kLean>
__global__ void __launch_bounds__(kGgsThreads, 1)
ggs_entry(const __grid_constant__ GgsBatch batch, const __grid_constant__ GgsParams P) {
  ggs_body<kEval, kPaired, kProbe, kLean>(batch.prob[blockIdx.x / P.ctas_per_problem], P);
}

// segs_fit: every CTA of every sequence in the batch touches at most kGgsMaxSeg segments (ggs_lean_fits)
template <bool kEval, bool kPaired, bool kProbe = false>
int launch_ggs_chunk(Context* ctx, const GgsBatch& batch, int nprob, int max_frames, long long max_rounds,
                     GgsParams P, bool segs_fit, cudaStream_t st) {
  if constexpr (!kEval && !kProbe) {  // the timing probe is its own instantiation (armed by pdb_debug_ggs_clocks, single-sequence calls)
    if (batch.prob[0].dbg_clock) return launch_ggs_chunk<kEval, kPaired, true>(ctx, batch, nprob, max_frames, max_rounds, P, segs_fit, st);
  }
  const int cpp = P.ctas_per_problem;  // ggs_plan
  // shared-memory match cache: everything beyond the fixed per-frame state, in rounds of 512 B
  const size_t fixed = ggs_smem_fixed_bytes(max_frames);
  const size_t budget = ctx->smem_optin > fixed + 1024 ? ctx->smem_optin - fixed - 1024 : 0;
  const long long rounds_per_cta = ggs_rounds_per_cta(max_rounds, cpp, kPaired);
  // PDB_GGS_FORCE_STREAM=1 disables the shared-memory-resident mode (tests exercise the streaming ring with it)
  const char* force_stream = getenv("PDB_GGS_FORCE_STREAM");
  const bool resident = (size_t)rounds_per_cta * 512 <= budget && !(force_stream && force_stream[0] == '1');
  P.resident_rounds = resident ? (int)rounds_per_cta : 0;
  P.ring = resident ? 0 : 1;
  // the lean instantiation serves the case it was specialised for; PDB_GGS_LEAN=0 keeps the general kernel (tests compare the two)
  const char* lean_env = getenv("PDB_GGS_LEAN");
  const bool lean = !kEval && resident && segs_fit && P.xch_mode == 1 && !(lean_env && lean_env[0] == '0');
  const void* kernel = lean ? (const void*)ggs_entry<kEval, kPaired, kProbe, !kEval> : (const void*)ggs_entry<kEval, kPaired, kProbe, false>;
  const size_t smem = fixed + (resident ? (size_t)rounds_per_cta * 512 : (size_t)kRingBytes);
  size_t& attr_bytes = ctx->attr->ggs[(kEval ? 1 : 0) + (kPaired ? 2 : 0) + (kProbe ? 4 : 0) + (lean ? 8 : 0)];
  if (smem > attr_bytes) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_bytes = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(cpp * nprob);
  cfg.blockDim = dim3(kGgsThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  {
    ScopedTimer timer(ctx, st, 0);
    void* args[] = {const_cast<GgsBatch*>(&batch), &P};
    PDB_CUDA(ctx, cudaLaunchKernelExC(&cfg, kernel, args));
  }
  ctx->launches += 1;
  return PDB_OK;
}

// All match sets of one launch share a stream layout (it is a property of the context they were packed on).
template <bool kEval>
int launch_ggs_layout(Context* ctx, int layout, const GgsBatch& batch, int nprob, int max_frames, long long max_rounds,
                      const GgsParams& P, bool segs_fit, cudaStream_t st) {
  if (layout == kLayoutPaired) return launch_ggs_chunk<kEval, true>(ctx, batch, nprob, max_frames, max_rounds, P, segs_fit, st);
  return launch_ggs_chunk<kEval, false>(ctx, batch, nprob, max_frames, max_rounds, P, segs_fit, st);
}
}  // namespace

namespace pdb {

// One match set per sequence, all packed for `frames` frames (the pose stride of pose_dev [batch, frames, 9]) and in one
// stream layout.  frames <= 0: take the frame count of the first set (pdb_ggs, whose pose shape is defined by the sets).
int check_ggs_problems(Context* ctx, pdb_matches* const* problems, int batch, int frames) {
  if (batch < 1 || !problems) return ctx->fail(PDB_ERR_INVALID, "bad GGS arguments");
  for (int b = 0; b < batch; ++b) {
    if (!problems[b]) return ctx->fail(PDB_ERR_INVALID, "null match set %d", b);
    const Matches* m = reinterpret_cast<const Matches*>(problems[b]);
    if (frames <= 0) frames = m->frames;
    if (m->frames != frames)
      return ctx->fail(PDB_ERR_INVALID, "match set %d was packed for %d frames (img_shape[0]), the pose has %d", b, m->frames, frames);
    if (m->layout != reinterpret_cast<const Matches*>(problems[0])->layout)
      return ctx->fail(PDB_ERR_INVALID, "all match sets of a batch must use the same stream layout (pdb_ggs_layout)");
  }
  return PDB_OK;
}

// Enqueue geometry-guided sampling for `batch` sequences (pose_dev [batch, frames, 9] updated in place).
int enqueue_ggs(Context* ctx, pdb_matches* const* problems, int batch, int frames, float* pose_dev, const pdb_ggs_config* cfg,
                pdb_ggs_stats* stats_dev, cudaStream_t st) {
  if (batch < 1 || !problems || !pose_dev || !cfg) return ctx->fail(PDB_ERR_INVALID, "bad GGS arguments");
  if (cfg->iter_num < 0) return ctx->fail(PDB_ERR_INVALID, "iter_num < 0");
  if (int rc = check_ggs_problems(ctx, problems, batch, frames)) return rc;
  int max_frames = 0;
  for (int b = 0; b < batch; ++b) {
    const Matches* m = reinterpret_cast<const Matches*>(problems[b]);
    max_frames = max_frames > m->frames ? max_frames : m->frames;
  }
  // exchange slots for every launch of this call (at most kGgsBatchMax sequences per launch): sized for the worst plan
  size_t ws_need = 0;
  for (int b0 = 0; b0 < batch; b0 += kGgsBatchMax) {
    const int nb = (batch - b0) < kGgsBatchMax ? (batch - b0) : kGgsBatchMax;
    long long max_rounds = 1;
    for (int i = 0; i < nb; ++i) {
      const Matches* m = reinterpret_cast<const Matches*>(problems[b0 + i]);
      max_rounds = max_rounds > m->rounds ? max_rounds : m->rounds;
    }
    int cpp, group;
    ggs_plan(ctx, nb, max_rounds, &cpp, &group);
    ws_need += (size_t)nb * ggs_ws_per_problem(max_frames, cpp, group);
  }
  if (int rc = ensure_buffer(ctx, &ctx->ggs_ws, &ctx->ggs_ws_bytes, ws_need)) return rc;
  PDB_CUDA(ctx, cudaMemsetAsync(ctx->ggs_ws, 0, ws_need, st));  // tags restart at 1 in every launch
  GgsParams P = {};
  P.n_phases = PDB_GGS_PHASES;
  const int n = cfg->iter_num;
  const int iters[PDB_GGS_PHASES] = {2 * n, n, n, n, 2 * n};           // :86-87
  const int flags[PDB_GGS_PHASES] = {7, 4, 1, 2, 7};                     // all | FL | R | T | all (:47-64)
  for (int i = 0; i < PDB_GGS_PHASES; ++i) {
    P.iters[i] = iters[i];
    P.flags[i] = flags[i];
  }
  P.alpha = (float)cfg->alpha;
  P.lr = (float)cfg->learning_rate;
  P.smax = (float)cfg->sampson_max;
  P.momentum = (float)cfg->momentum;
  P.min_matches = cfg->min_matches;
  const int N = max_frames;
  char* ws = static_cast<char*>(ctx->ggs_ws);
  for (int b0 = 0; b0 < batch; b0 += kGgsBatchMax) {
    const int nb = (batch - b0) < kGgsBatchMax ? (batch - b0) : kGgsBatchMax;
    GgsBatch gb = {};
    long long max_rounds = 1;
    for (int i = 0; i < nb; ++i) {
      const Matches* m = reinterpret_cast<const Matches*>(problems[b0 + i]);
      max_rounds = max_rounds > m->rounds ? max_rounds : m->rounds;
    }
    ggs_plan(ctx, nb, max_rounds, &P.ctas_per_problem, &P.xch_group);
    P.xch_mode = ggs_xch_mode();
    bool segs_fit = true;
    for (int i = 0; i < nb; ++i) {
      const Matches* m = reinterpret_cast<const Matches*>(problems[b0 + i]);
      segs_fit = segs_fit && ggs_lean_fits(m->host_segs.data(), m->nseg, m->rounds, P.ctas_per_problem, m->layout == kLayoutPaired);
      GgsProblem& p = gb.prob[i];
      p.pts = m->pts;
      p.segs = m->segs;
      p.nseg = m->nseg;
      p.rounds = m->rounds;
      p.m_total = m->m_total;
      p.frames = m->frames;
      p.height = (float)m->height;
      p.width = (float)m->width;
      p.pose = pose_dev + (size_t)(b0 + i) * N * 9;
      p.xch1 = reinterpret_cast<unsigned long long*>(ws);
      p.xch2 = p.xch1 + 2 * (size_t)P.ctas_per_problem * ggs_xch_words(m->frames);
      p.acc = reinterpret_cast<float*>(ws + ggs_ws_slots_bytes(max_frames, P.ctas_per_problem, P.xch_group));
      p.stats = stats_dev ? stats_dev + (b0 + i) : nullptr;
      p.dbg_clock = (ctx->ggs_clock && !ctx->den_clock && batch == 1) ? ctx->ggs_clock : nullptr;
      ws += ggs_ws_per_problem(max_frames, P.ctas_per_problem, P.xch_group);
    }
    const int layout = reinterpret_cast<const Matches*>(problems[b0])->layout;
    if (int rc = launch_ggs_layout<false>(ctx, layout, gb, nb, max_frames, max_rounds, P, segs_fit, st)) return rc;
  }
  return PDB_OK;
}

}  // namespace pdb

extern "C" {

int pdb_ggs(pdb_context* c, pdb_matches* const* problems, int32_t batch, float* pose_dev, const pdb_ggs_config* cfg,
            pdb_ggs_stats* stats_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  return enqueue_ggs(ctx, problems, batch, 0, pose_dev, cfg, stats_dev, static_cast<cudaStream_t>(stream));
}

int pdb_sampson_eval(pdb_context* c, const pdb_matches* pm, const float* pose_dev, int32_t update_R, int32_t update_T,
                     int32_t update_FL, double sampson_max, float* grad_dev, float* scalars_dev, float* F_dev,
                     float* G_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!pm || !pose_dev || !grad_dev || !scalars_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  const Matches* m = reinterpret_cast<const Matches*>(pm);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  GgsParams P = {};
  ggs_plan(ctx, 1, m->rounds > 0 ? m->rounds : 1, &P.ctas_per_problem, &P.xch_group);
  P.xch_mode = ggs_xch_mode();
  const size_t ws_need = ggs_ws_per_problem(m->frames, P.ctas_per_problem, P.xch_group);
  if (int rc = ensure_buffer(ctx, &ctx->ggs_ws, &ctx->ggs_ws_bytes, ws_need)) return rc;
  PDB_CUDA(ctx, cudaMemsetAsync(ctx->ggs_ws, 0, ws_need, st));
  if (G_dev) PDB_CUDA(ctx, cudaMemsetAsync(G_dev, 0, sizeof(float) * 9 * (m->nseg ? m->nseg : 1), st));
  P.n_phases = 1;
  P.iters[0] = 1;
  P.flags[0] = (update_R ? 1 : 0) | (update_T ? 2 : 0) | (update_FL ? 4 : 0);
  P.alpha = 1e-4f;
  P.lr = 1e-2f;
  P.smax = (float)sampson_max;
  P.momentum = 0.9f;
  P.min_matches = 0.0;
  GgsBatch gb = {};
  GgsProblem& p = gb.prob[0];
  char* ws = static_cast<char*>(ctx->ggs_ws);
  p.pts = m->pts;
  p.segs = m->segs;
  p.nseg = m->nseg;
  p.rounds = m->rounds;
  p.m_total = m->m_total;
  p.frames = m->frames;
  p.height = (float)m->height;
  p.width = (float)m->width;
  p.pose = const_cast<float*>(pose_dev);  // eval mode never writes the pose
  p.xch1 = reinterpret_cast<unsigned long long*>(ws);
  p.xch2 = p.xch1 + 2 * (size_t)P.ctas_per_problem * ggs_xch_words(m->frames);
  p.acc = reinterpret_cast<float*>(ws + ggs_ws_slots_bytes(m->frames, P.ctas_per_problem, P.xch_group));
  p.dbg_grad = grad_dev;
  p.dbg_scalars = scalars_dev;
  p.dbg_F = F_dev;
  p.dbg_G = G_dev;
  return launch_ggs_layout<true>(ctx, m->layout, gb, 1, m->frames, m->rounds > 0 ? m->rounds : 1, P, false, st);
}

}  // extern "C"
