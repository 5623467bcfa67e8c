// Layout of the packed match stream (pdb_matches) and the static work partition of the GGS kernel.
// Host + device: the packer (api_core.cu), the kernel (ggs.cuh) and the CPU harness (tests/host/geom_host.cu) all use
// exactly these functions, so the layout contract can be checked without a GPU.
//
//   plain  : one float4 (u1,v1,u2,v2) per match; a pair segment occupies ceil(count/32) ROUNDS of 32 rows (512 B, one
//            coalesced warp load); padding rows are zero.
//   paired : a pair segment occupies whole UNITS of two rounds (64 rows, 1 KB).  Inside unit U lane l owns two matches,
//            A = row 64 U + l and B = row 64 U + 32 + l of the plain order, stored component-interleaved:
//                pts[64 U + l]      = (u1_A, u1_B, v1_A, v1_B)
//                pts[64 U + 32 + l] = (u2_A, u2_B, v2_A, v2_B)
//            so that the two 128-bit loads of a lane hold the two matches' operands side by side (sampson_match2_unit
//            in ggs.cuh); with the plain layout the compiler re-pairs the components of two float4 with extra MOVs.
//            Every segment starts at an even round and all partition boundaries are even, so a unit never straddles
//            two segments, two warps or two CTAs.
#pragma once
#include "geom.cuh"

namespace pdb {

enum : int { kLayoutPlain = 0, kLayoutPaired = 1 };

// rounds of 32 rows a segment of `count` matches occupies
PDB_HD long long layout_seg_rounds(long long count, bool paired) {
  return paired ? (count + 63) / 64 * 2 : (count + 31) / 32;
}

// Index, in the float view of pts, of component `comp` (0 u1, 1 v1, 2 u2, 3 v2) of the k-th match of a segment that
// starts at round `first_round`.
PDB_HD size_t layout_float_index(long long first_round, long long k, int comp, bool paired) {
  if (!paired) return ((size_t)first_round * 32 + (size_t)k) * 4 + (size_t)comp;
  const long long unit = k >> 6;
  const int within = (int)(k & 63), half = within >> 5, lane = within & 31;
  const size_t quad = (size_t)first_round * 32 + (size_t)unit * 64 + (size_t)(comp >> 1) * 32 + (size_t)lane;
  return quad * 4 + (size_t)((comp & 1) * 2 + half);
}

// rounds [r0, r1) of CTA `cta` out of `cpp` CTAs that share a match set of `rounds` rounds
PDB_HD void ggs_cta_range(long long rounds, int cta, int cpp, bool paired, int* r0, int* r1) {
  if (paired) {
    const long long units = rounds >> 1;
    *r0 = 2 * (int)(units * cta / cpp);
    *r1 = 2 * (int)(units * (cta + 1) / cpp);
  } else {
    *r0 = (int)(rounds * cta / cpp);
    *r1 = (int)(rounds * (cta + 1) / cpp);
  }
}

// rounds [r0, r1) of warp `warp` out of `nwarps` inside the CTA range [r_cta0, r_cta1)
PDB_HD void ggs_warp_range(int r_cta0, int r_cta1, int warp, int nwarps, bool paired, int* r0, int* r1) {
  if (paired) {
    const long long units = (r_cta1 - r_cta0) >> 1;
    *r0 = r_cta0 + 2 * (int)(units * warp / nwarps);
    *r1 = r_cta0 + 2 * (int)(units * (warp + 1) / nwarps);
  } else {
    *r0 = r_cta0 + (int)((long long)(r_cta1 - r_cta0) * warp / nwarps);
    *r1 = r_cta0 + (int)((long long)(r_cta1 - r_cta0) * (warp + 1) / nwarps);
  }
}

// Segment-aware warp partition: rounds [r0, r1) of warp `warp` inside the CTA range [r_cta0, r_cta1), which intersects the pair
// segments seg_lo..seg_hi (segs[s].x = first round of segment s; segs[nseg].x = total rounds).  The CTA's warps are first
// distributed over those segments -- one each, the rest greedily to the segment with the largest share per warp -- and the
// part of a segment inside the CTA is then split evenly among its warps, so that NO warp crosses a segment boundary: every
// (warp, segment) visit costs an F' set-up and a 16-shuffle reduction, and the warps that paid two of them were the stragglers
// of stage 1.  Falls back to the even split when the CTA touches more segments than it has warps.
PDB_HD void ggs_warp_range_seg(const int4* segs, int seg_lo, int seg_hi, int r_cta0, int r_cta1, int warp, int nwarps, bool paired,
                               int* r0, int* r1) {
  const int nseg_c = seg_hi - seg_lo + 1;
  if (r_cta1 <= r_cta0 || nseg_c < 1 || nseg_c > nwarps || nwarps > 16) {
    ggs_warp_range(r_cta0, r_cta1, warp, nwarps, paired, r0, r1);
    return;
  }
  const int g = paired ? 2 : 1;  // granule: whole units in the paired layout (segments and CTA ranges start on even rounds)
  int share[16], wcount[16];
  for (int k = 0; k < nseg_c; ++k) {
    const int lo = segs[seg_lo + k].x > r_cta0 ? segs[seg_lo + k].x : r_cta0;
    const int hi = segs[seg_lo + k + 1].x < r_cta1 ? segs[seg_lo + k + 1].x : r_cta1;
    share[k] = (hi - lo) / g;
    wcount[k] = 1;
  }
  for (int extra = nwarps - nseg_c; extra > 0; --extra) {  // next warp to the segment with the largest share per warp (first wins ties)
    int best = 0;
    for (int k = 1; k < nseg_c; ++k)
      if ((long long)share[k] * wcount[best] > (long long)share[best] * wcount[k]) best = k;
    wcount[best] += 1;
  }
  int k = 0, base = 0;
  while (warp >= base + wcount[k]) base += wcount[k++];
  const int idx = warp - base;
  const int lo = segs[seg_lo + k].x > r_cta0 ? segs[seg_lo + k].x : r_cta0;
  *r0 = lo + g * (int)((long long)share[k] * idx / wcount[k]);
  *r1 = lo + g * (int)((long long)share[k] * (idx + 1) / wcount[k]);
}

// upper bound of the rounds one CTA can own (sizes the shared-memory match cache)
PDB_HD long long ggs_rounds_per_cta(long long max_rounds, int cpp, bool paired) {
  if (paired) return 2 * (((max_rounds >> 1) + cpp - 1) / cpp);
  return (max_rounds + cpp - 1) / cpp + 1;
}

// The two matches of a lane inside a paired unit, in the plain component order (u1, v1, u2, v2).
PDB_HD float4 unit_match_a(const float4 X, const float4 Y) { return make_float4(X.x, X.z, Y.x, Y.z); }
PDB_HD float4 unit_match_b(const float4 X, const float4 Y) { return make_float4(X.y, X.w, Y.y, Y.w); }

}  // namespace pdb
