// The map hash grid's cell keys and probes, shared by the scan-to-map search (mapping.cu) and every prior-map or keyframe inlier
// score (reloc.cu: k_reloc_score, k_inlier_score): all must find a point's cell under the same key and hash.  Every score picks
// its points with scoring_point / scoring_points and counts a warp's moved points with warp_inliers, so scores of one pose taken
// by different kernels are equal (recovery compares a candidate's k_reloc_score count with its row's k_inlier_score count).
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

// the scoring points of stacks of n_c corner and n_s surf points: at most max_pts of each type, m_c = min(n_c, max_pts) corner
// points first
__device__ __forceinline__ int scoring_points(int n_c, int n_s, int max_pts) { return min(n_c, max_pts) + min(n_s, max_pts); }

// scoring point i (< m_c + m_s): corner stack point floor(i n_c / m_c), or surf stack point floor((i - m_c) n_s / m_s)
__device__ __forceinline__ float4 scoring_point(const Pt4* __restrict__ corner, const Pt4* __restrict__ surf, int n_c, int m_c, int n_s, int m_s, int i) {
  const Pt4 p = i < m_c ? corner[(long long)i * n_c / m_c] : surf[(long long)(i - m_c) * n_s / m_s];
  return make_float4(p.x, p.y, p.z, p.i);
}

// cnt plus the inliers among scoring points p0 .. p0 + np - 1 (np <= 32) once moved: lane j holds point p0 + j at (qx, qy, qz);
// points below m_c are corner points.  The warp walks the points in turn, each through any_in_block27 over its type's grid (mask:
// the grid's dyn->mask, hoisted by the caller), and a point is an inlier when some map point lies at float d2 < inlier_sq: it
// needs a map point, not the nearest one.  Warp-uniform; every lane takes part and gets the count.  (The running count goes in
// rather than being added to the result: k_reloc_score then keeps its 55 registers.)
__device__ __forceinline__ int warp_inliers(int cnt, float qx, float qy, float qz, int p0, int np, int m_c, const GridTable& corner,
                                            unsigned mask_c, const GridTable& surf, unsigned mask_s, float inlier_sq) {
  for (int j = 0; j < np; ++j) {
    const float px = __shfl_sync(0xffffffffu, qx, j), py = __shfl_sync(0xffffffffu, qy, j), pz = __shfl_sync(0xffffffffu, qz, j);
    const bool is_corner = p0 + j < m_c;
    const bool in = any_in_block27(is_corner ? corner : surf, is_corner ? mask_c : mask_s, px, py, pz,
                                   [&](float u, float v, float w) { return sqdist3(u, v, w, px, py, pz) < inlier_sq; });
    cnt += in ? 1 : 0;
  }
  return cnt;
}

}  // namespace aloam
