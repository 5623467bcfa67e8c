// Image preprocessing entry (load_and_preprocess_images, util/load_img_folder.py): decoded uint8 HWC frames on the host ->
// float32 [n,3,S,S] on the device.  Bilinear downsampling without antialias reads at most two source rows per output row, so
// per frame only those rows' crop columns are uploaded (a 1066-wide crop resized to 224 touches at most 448 of its 1066 rows).
// They are gathered from the caller's pageable arrays into one of two pinned slots while the other slot's upload is in flight;
// each frame's kernel follows its upload on the stream.
#include <climits>
#include <cstring>
#include <vector>

#include "context.cuh"
#include "preprocess.cuh"

using namespace pdb;

namespace {

size_t round16(size_t v) { return (v + 15) & ~(size_t)15; }

}  // namespace

extern "C" int pdb_images_preprocess_host(pdb_context* c, int32_t n, const uint8_t* const* rgb_host, const int32_t* hw,
                                          const int32_t* crop, int32_t out_size, float* images_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (n <= 0) return ctx->fail(PDB_ERR_INVALID, "n = %d frames", n);
  if (out_size <= 0) return ctx->fail(PDB_ERR_INVALID, "out_size = %d", out_size);
  if (!rgb_host || !hw || !crop || !images_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if ((long long)out_size * out_size > INT_MAX) return ctx->fail(PDB_ERR_LIMIT, "out_size %d: too many pixels per frame", out_size);
  const int S = out_size;
  for (int i = 0; i < n; ++i) {
    const long long H = hw[2 * i], W = hw[2 * i + 1], top = crop[3 * i], left = crop[3 * i + 1], side = crop[3 * i + 2];
    if (!rgb_host[i]) return ctx->fail(PDB_ERR_INVALID, "frame %d: null pixels", i);
    if (side < 2 || top < 0 || left < 0 || top + side > H || left + side > W)
      return ctx->fail(PDB_ERR_INVALID, "frame %d: crop (top %lld, left %lld, side %lld) outside the %lldx%lld image or side < 2", i,
                       top, left, side, H, W);
  }
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  // plans: the row map and the staged crop rows of every frame, and where each frame's region lies in the device buffer
  std::vector<int2> maps((size_t)n * S);
  std::vector<std::vector<int>> rows(n);
  std::vector<size_t> off(n + 1, 0);
  std::vector<int> compact;
  size_t slot_need = 0;
  for (int i = 0; i < n; ++i) {
    const int side = crop[3 * i + 2];
    compact.resize(side);
    rows[i].resize(side);
    rows[i].resize(pre_plan(side, S, compact.data(), &maps[(size_t)i * S], rows[i].data()));
    const size_t bytes = round16(pre_map_bytes(S) + rows[i].size() * 3 * (size_t)side);
    off[i + 1] = off[i] + bytes;
    if (bytes > slot_need) slot_need = bytes;
  }
  if (int rc = ensure_buffer(ctx, &ctx->pre_dev, &ctx->pre_dev_bytes, off[n])) return rc;
  for (int s = 0; s < 2; ++s) {
    if (ctx->pre_pin_bytes[s] < slot_need) {  // the previous call synchronised: no upload reads the old slot
      if (ctx->pre_pin[s]) cudaFreeHost(ctx->pre_pin[s]);
      ctx->pre_pin[s] = nullptr;
      ctx->pre_pin_bytes[s] = 0;
      PDB_CUDA(ctx, cudaHostAlloc(&ctx->pre_pin[s], slot_need + slot_need / 4, cudaHostAllocDefault));
      ctx->pre_pin_bytes[s] = slot_need + slot_need / 4;
    }
    if (!ctx->pre_ev[s]) PDB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->pre_ev[s], cudaEventDisableTiming));
  }

  uint8_t* dev = static_cast<uint8_t*>(ctx->pre_dev);
  for (int i = 0; i < n; ++i) {
    const int slot = i & 1, W = hw[2 * i + 1], top = crop[3 * i], left = crop[3 * i + 1], side = crop[3 * i + 2];
    PDB_CUDA(ctx, cudaEventSynchronize(ctx->pre_ev[slot]));  // the upload of frame i-2 has left this slot
    uint8_t* h = static_cast<uint8_t*>(ctx->pre_pin[slot]);
    memcpy(h, &maps[(size_t)i * S], sizeof(int2) * S);
    const size_t pitch = (size_t)3 * side;
    uint8_t* dst = h + pre_map_bytes(S);
    for (size_t k = 0; k < rows[i].size(); ++k)
      memcpy(dst + k * pitch, rgb_host[i] + ((size_t)(top + rows[i][k]) * W + left) * 3, pitch);
    PDB_CUDA(ctx, cudaMemcpyAsync(dev + off[i], h, off[i + 1] - off[i], cudaMemcpyHostToDevice, st));
    PDB_CUDA(ctx, cudaEventRecord(ctx->pre_ev[slot], st));
    preprocess_kernel<<<(S * S + 255) / 256, 256, 0, st>>>(dev + off[i], side, S, images_dev + (size_t)i * 3 * S * S);
    PDB_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
  }
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  return PDB_OK;
}
