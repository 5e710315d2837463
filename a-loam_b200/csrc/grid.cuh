// The map hash grid's cell keys and probes, shared by the scan-to-map search (mapping.cu), the relocaliser's scoring (reloc.cu)
// and the tracking score of per-row records (rows.cu): all must find a point's cell under the same key and hash, and the two
// scores must pick and test their points alike.
#pragma once
#include "kernels.h"

namespace aloam {

constexpr unsigned long long kEmpty = ~0ull;

__device__ __forceinline__ unsigned long long cell_key(int cx, int cy, int cz) {
  return ((unsigned long long)(unsigned)(cx + (1 << 20)) << 42) | ((unsigned long long)(unsigned)(cy + (1 << 20)) << 21) |
         (unsigned long long)(unsigned)(cz + (1 << 20));
}
__device__ __forceinline__ unsigned hash_key(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (unsigned)k;
}
__device__ __forceinline__ int cell_of(float v, float inv_cs) { return (int)floorf(v * inv_cs); }
__device__ __forceinline__ unsigned long long slot_key(const uint4& s) { return ((unsigned long long)s.y << 32) | s.x; }

__device__ __forceinline__ int warp_incl_scan(int v) {
  const unsigned lane = lane_id();
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= (unsigned)d) v += t;
  }
  return v;
}

// The 27 cells around q as visit_block27 (mapping.cu) walks them, with an exit: true as soon as a chunk of 32 candidates holds
// one for which pred(x, y, z) is true, false when no candidate does.  Warp-uniform; every lane takes part.
template <typename P>
__device__ __forceinline__ bool any_in_block27(const GridTable& g, unsigned mask, float qx, float qy, float qz, P&& pred) {
  const int lane = (int)lane_id();
  const int cx = cell_of(qx, g.inv_cs), cy = cell_of(qy, g.inv_cs), cz = cell_of(qz, g.inv_cs);
  int start = 0, cnt = 0;
  if (lane < 27) {
    const int dz = lane / 9 - 1, dy = (lane % 9) / 3 - 1, dx = lane % 3 - 1;
    const unsigned long long key = cell_key(cx + dx, cy + dy, cz + dz);
    unsigned h = hash_key(key) & mask;
    for (;;) {
      const uint4 s = __ldg(g.slots + h);
      const unsigned long long k = slot_key(s);
      if (k == key) { cnt = (int)s.z; start = (int)s.w - cnt; break; }
      if (k == kEmpty) break;
      h = (h + 1) & mask;
    }
  }
  const int incl = warp_incl_scan(cnt);
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  for (int e0 = 0; e0 < total; e0 += 32) {
    const int e = e0 + lane;
    int c = 0;
#pragma unroll
    for (int step = 16; step >= 1; step >>= 1) {
      const int v = __shfl_sync(0xffffffffu, incl, c + step - 1);
      if (v <= e) c += step;
    }
    c = min(c, 31);
    const int c_incl = __shfl_sync(0xffffffffu, incl, c);
    const int c_cnt = __shfl_sync(0xffffffffu, cnt, c);
    const int c_start = __shfl_sync(0xffffffffu, start, c);
    bool hit = false;
    if (e < total) {
      const float4 p = __ldg(g.gpts + c_start + (e - (c_incl - c_cnt)));
      hit = pred(p.x, p.y, p.z);
    }
    if (__any_sync(0xffffffffu, hit)) return true;
  }
  return false;
}

// scoring point i (< m_c + m_s): corner stack point floor(i n_c / m_c), or surf stack point floor((i - m_c) n_s / m_s)
__device__ __forceinline__ float4 scoring_point(const Pt4* __restrict__ corner, const Pt4* __restrict__ surf, int n_c, int m_c, int n_s, int m_s, int i) {
  const Pt4 p = i < m_c ? corner[(long long)i * n_c / m_c] : surf[(long long)(i - m_c) * n_s / m_s];
  return make_float4(p.x, p.y, p.z, p.i);
}

}  // namespace aloam
