// TEST HARNESS (not product): posediffusion_b200/csrc/preprocess.cuh on the CPU.  The staging planner and the kernel body
// (pre_pixel, what preprocess_kernel runs per thread) execute sequentially over the same staging layout that
// pdb_images_preprocess_host uploads, so the CPU tests check the planner's row set and the kernel's arithmetic against the
// reference fixtures without a GPU.
#include <cstring>
#include <vector>

#include "../../posediffusion_b200/csrc/preprocess.cuh"

using namespace pdb;

// Rows the kernel reads for output rows 0..S-1 of a crop of `side` rows that the plan does not stage at the compact index the
// row map names (0 = the plan covers every read).  rows_out [side] receives the staged crop rows, *count_out their number.
extern "C" int pre_host_plan_misses(int side, int S, int* rows_out, int* count_out) {
  std::vector<int> compact(side);
  std::vector<int2> map(S);
  const int count = pre_plan(side, S, compact.data(), map.data(), rows_out);
  *count_out = count;
  int misses = 0;
  for (int y = 0; y < S; ++y) {
    const PreTap t = pre_tap(y, side, S);
    const int2 m = map[y];
    if (m.x < 0 || m.x >= count || rows_out[m.x] != t.i0) ++misses;
    if (m.y < 0 || m.y >= count || rows_out[m.y] != t.i1) ++misses;
  }
  return misses;
}

extern "C" void pre_host_tap(int dst, int in, int out, int* i01, float* l01) {
  const PreTap t = pre_tap(dst, in, out);
  i01[0] = t.i0;
  i01[1] = t.i1;
  l01[0] = t.l0;
  l01[1] = t.l1;
}

// pdb_images_preprocess_host without the device: plan, gather the touched crop rows into a staging region, run the kernel body
// for every output pixel.  out [n,3,S,S].
extern "C" int pre_host_run(int n, const uint8_t* const* rgb, const int* hw, const int* crop, int S, float* out) {
  for (int i = 0; i < n; ++i) {
    const int W = hw[2 * i + 1], top = crop[3 * i], left = crop[3 * i + 1], side = crop[3 * i + 2];
    std::vector<int> compact(side), rows(side);
    std::vector<int2> map(S);
    const int count = pre_plan(side, S, compact.data(), map.data(), rows.data());
    const size_t pitch = (size_t)3 * side;
    std::vector<uint8_t> stage(pre_map_bytes(S) + count * pitch);
    memcpy(stage.data(), map.data(), sizeof(int2) * S);
    for (int k = 0; k < count; ++k)
      memcpy(stage.data() + pre_map_bytes(S) + k * pitch, rgb[i] + ((size_t)(top + rows[k]) * W + left) * 3, pitch);
    float* o = out + (size_t)i * 3 * S * S;
    for (int y = 0; y < S; ++y)
      for (int x = 0; x < S; ++x) pre_pixel(stage.data(), side, S, x, y, o);
  }
  return 0;
}
