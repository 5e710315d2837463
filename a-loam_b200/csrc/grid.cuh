// The map hash grid's cell keys and probes, shared by the scan-to-map search (mapping.cu) and the relocaliser's scoring
// (reloc.cu): both must find a point's cell under the same key and hash.
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

}  // namespace aloam
