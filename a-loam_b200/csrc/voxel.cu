// pcl::VoxelGrid<PointXYZI>::applyFilter as one segmented, device-resident GPU routine: S independent clouds ("segments",
// each with its own leaf size) are filtered by ONE sequence of launches -- a single cloud (aloam_voxel_filter), the two scan
// stacks of a mapping frame (laserMapping.cpp:543-549, downSizeFilterCorner / downSizeFilterSurf), or all valid cubes of the
// map after insertion (:787-801, up to 75 corner + 75 surf cubes).  The per-ring 0.2 m instance of scanRegistration.cpp:401-407
// is fused into k_ring_features.  Semantics per SURVEY.md 8a "V", per segment:
//   bounding box -> min_b / div_b -> voxel index (float multiply, floor) -> sort by index -> one output per occupied
//   voxel in ascending index order = float32 centroid of x, y, z, intensity accumulated in sorted order.
// Key = segment << idx_bits | voxel index (PCL's index inside the segment's own bounding box), so one stable LSD radix sort
// (8 bits per pass) orders every segment by voxel and keeps the segments apart.  PCL's std::sort is unstable; here ties are
// resolved by point index, which is the CANONICAL order of the oracle.  Sizes live in device memory; nothing here
// synchronises with the host.  A segment whose index range overflows int (PCL: "leaf size is too small", input returned
// unchanged) or idx_bits (flagged) is returned as it is: its key is the position and the write-back copies the source.
#include <climits>
#include <cfloat>
#include <cooperative_groups.h>
#include "ctx.h"

namespace aloam {

namespace {
constexpr int VT = 256, VCH = 1024, VIT = VCH / VT;

__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : (i ^ 0x7fffffff); }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : (i ^ 0x7fffffff)); }
}  // namespace

// All passes of the LSD radix sort in ONE cooperative launch (the segmented filters of the mapper sort a few 10^4 keys: twelve
// launches of a few microseconds each were launch latency, not work).  Tiles of VCH keys go round-robin over the CTAs; per pass:
// tile histograms -> grid barrier -> every CTA derives the offsets of its own tiles from the histogram table (thread = digit:
// digit totals over all tiles, block-wide exclusive scan, plus the running sum over the tiles before its own) and scatters ->
// grid barrier.  Within a digit the keys keep their order (stable); the result is in buffer (passes & 1).
__device__ __forceinline__ void radix_sort_all_body(unsigned* __restrict__ k0, int* __restrict__ v0, unsigned* __restrict__ k1, int* __restrict__ v1,
                                                       const int* __restrict__ n_ptr, int bits, int* __restrict__ hist) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ int s_h[256];
  __shared__ int s_w[VT / 32];
  __shared__ int s_cnt[VIT * (VT / 32)][256];
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int n = *n_ptr;
  const int tiles = (n + VCH - 1) / VCH;
  int cur = 0;
  for (int shift = 0; shift < bits; shift += 8) {   // `bits` is a launch parameter: every CTA passes the same barriers
    const unsigned* __restrict__ kin = cur ? k1 : k0;
    const int* __restrict__ vin = cur ? v1 : v0;
    unsigned* __restrict__ kout = cur ? k0 : k1;
    int* __restrict__ vout = cur ? v0 : v1;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      s_h[tid] = 0;
      __syncthreads();
#pragma unroll
      for (int it = 0; it < VIT; ++it) {
        const int i = t * VCH + it * VT + tid;
        if (i < n) atomicAdd(&s_h[(kin[i] >> shift) & 255u], 1);
      }
      __syncthreads();
      hist[t * 256 + tid] = s_h[tid];
      __syncthreads();
    }
    grid.sync();
    // thread = digit: start of the digit in the output = exclusive scan of the digit totals
    int tot = 0, pre = 0, pre_upto = 0;   // pre = sum of hist[t'][digit] over the tiles t' < pre_upto
    for (int t = 0; t < tiles; ++t) tot += hist[t * 256 + tid];
    int incl = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
    if (lane == 31) s_w[w] = incl;
    __syncthreads();
    int wb = 0;
    for (int k = 0; k < w; ++k) wb += s_w[k];
    const int start = wb + incl - tot;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      for (; pre_upto < t; ++pre_upto) pre += hist[pre_upto * 256 + tid];
      for (int k = tid; k < VIT * (VT / 32) * 256; k += VT) (&s_cnt[0][0])[k] = 0;
      __syncthreads();
      int dig[VIT], rank[VIT];
#pragma unroll
      for (int it = 0; it < VIT; ++it) {
        const int i = t * VCH + it * VT + tid;
        const int d = i < n ? (int)((kin[i] >> shift) & 255u) : -1;
        dig[it] = d;
        const unsigned grp = __match_any_sync(0xffffffffu, d);
        rank[it] = __popc(grp & ((1u << lane) - 1u));
        if (d >= 0 && rank[it] == 0) s_cnt[it * (VT / 32) + w][d] = __popc(grp);
      }
      __syncthreads();
      {
        int run = start + pre;
#pragma unroll
        for (int k = 0; k < VIT * (VT / 32); ++k) { const int c = s_cnt[k][tid]; s_cnt[k][tid] = run; run += c; }
      }
      __syncthreads();
#pragma unroll
      for (int it = 0; it < VIT; ++it) {
        if (dig[it] < 0) continue;
        const int i = t * VCH + it * VT + tid;
        const int dst = s_cnt[it * (VT / 32) + w][dig[it]] + rank[it];
        kout[dst] = kin[i];
        vout[dst] = vin[i];
      }
      __syncthreads();
    }
    grid.sync();
    cur ^= 1;
  }
}
// grid (CTAs per lane, 1, lanes), cooperative: every lane sorts its own keys with its own tiles and histograms; the grid barriers
// span all lanes, which all run the same `bits` passes
__global__ void __launch_bounds__(VT) k_radix_sort_all(const __grid_constant__ Batch<VoxLane> B, int bits) {
  const VoxLane& a = B.a[blockIdx.z];
  radix_sort_all_body(a.keys[0], a.vals[0], a.keys[1], a.vals[1], a.f.total, bits, a.hist);
}
// one key array of any size (the prior-map build, cubemap.cu): the same passes over *n keys
__global__ void __launch_bounds__(VT) k_radix_sort_flat(unsigned* k0, int* v0, unsigned* k1, int* v1, const int* n, int bits, int* hist) {
  radix_sort_all_body(k0, v0, k1, v1, n, bits, hist);
}


// number of voxel heads (first element of each run of equal keys) per block of VCH sorted elements; the CTAs stride over
// the blocks, so the grid may be smaller than the live block count
__device__ __forceinline__ void vox_heads_body(const unsigned* __restrict__ keys, const int* __restrict__ n_ptr, int* __restrict__ block_heads) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int n = *n_ptr;
  __shared__ int s_c;
  for (int blk = blockIdx.x; blk * VCH < n; blk += gridDim.x) {
    if (threadIdx.x == 0) s_c = 0;
    __syncthreads();
    int c = 0;
#pragma unroll
    for (int it = 0; it < VIT; ++it) {
      const int i = blk * VCH + it * VT + threadIdx.x;
      if (i < n && (i == 0 || keys[i] != keys[i - 1])) ++c;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_c, c);
    __syncthreads();
    if (threadIdx.x == 0) block_heads[blk] = s_c;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(VT) k_vox_heads(const __grid_constant__ Batch<VoxLane> B, int cur) {
  const VoxLane& a = B.a[blockIdx.z];
  vox_heads_body(a.keys[cur], a.f.total, a.block_heads);
}


__device__ __forceinline__ void vox_blockscan_body(int* __restrict__ block_heads, const int* __restrict__ n_ptr, int* __restrict__ total) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int nblocks = (*n_ptr + VCH - 1) / VCH;
  __shared__ int s_w[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int per = (nblocks + 1023) / 1024;
  int sum = 0;
  for (int k = 0; k < per; ++k) { const int b = t * per + k; if (b < nblocks) sum += block_heads[b]; }
  int incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
  if (lane == 31) s_w[w] = incl;
  __syncthreads();
  if (w == 0) {
    int x = s_w[lane], inc = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += u; }
    s_w[lane] = inc - x;
    if (lane == 31) *total = inc;
  }
  __syncthreads();
  int run = s_w[w] + incl - sum;
  for (int k = 0; k < per; ++k) { const int b = t * per + k; if (b < nblocks) { const int c = block_heads[b]; block_heads[b] = run; run += c; } }
}
__global__ void __launch_bounds__(1024) k_vox_blockscan(const __grid_constant__ Batch<VoxLane> B) {
  const VoxLane& a = B.a[blockIdx.z];
  vox_blockscan_body(a.block_heads, a.f.total, a.heads_total);
}


__device__ __forceinline__ int seg_count(const SegFilter& f) { return min(max(*f.n_seg - f.seg0, 0), f.seg_cap); }
// segment number of a key; idx_bits may be 32 (one segment), so the shift is done in 64 bits
__device__ __forceinline__ int seg_of(unsigned key, int idx_bits) { return (int)((unsigned long long)key >> idx_bits); }

__device__ __forceinline__ void seg_prep_body(SegFilter f) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  __shared__ int s_w[8];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int S = seg_count(f);
  const int n = t < S ? max(0, *f.seg[f.seg0 + t].n_in) : 0;
  int incl = n;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
  if (lane == 31) s_w[w] = incl;
  __syncthreads();
  int base = 0;
  for (int v = 0; v < w; ++v) base += s_w[v];
  if (t <= ALOAM_MAX_SEGS) f.off[t] = 0;
  __syncthreads();
  if (t < S) f.off[t] = base + incl - n;
  if (t == S - 1 || (S == 0 && t == 0)) {
    const int total = S == 0 ? 0 : base + incl;
    for (int v = max(S, 0); v <= ALOAM_MAX_SEGS; ++v) f.off[v] = total;
    *f.total = total;
  }
  if (t < ALOAM_MAX_SEGS) {
    f.bbox[6 * t + 0] = INT_MAX; f.bbox[6 * t + 1] = INT_MAX; f.bbox[6 * t + 2] = INT_MAX;
    f.bbox[6 * t + 3] = INT_MIN; f.bbox[6 * t + 4] = INT_MIN; f.bbox[6 * t + 5] = INT_MIN;
  }
}
__global__ void __launch_bounds__(256) k_seg_prep(const __grid_constant__ Batch<VoxLane> B) { seg_prep_body(B.a[blockIdx.z].f); }


// grid (chunks, segments)
__device__ __forceinline__ void seg_bbox_body(SegFilter f) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int sgm = blockIdx.y;
  if (sgm >= seg_count(f)) return;
  const SegDesc d = f.seg[f.seg0 + sgm];
  const int n = *d.n_in;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  bool any = false;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const Pt4 p = d.src[i];
    lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
    hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
    any = true;
  }
  if (!__any_sync(0xffffffffu, any)) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int dd = 16; dd > 0; dd >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], dd));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], dd));
    }
    if ((threadIdx.x & 31) == 0) { atomicMin(&f.bbox[6 * sgm + a], f2ord(lo[a])); atomicMax(&f.bbox[6 * sgm + 3 + a], f2ord(hi[a])); }
  }
}
__global__ void __launch_bounds__(256) k_seg_bbox(const __grid_constant__ Batch<VoxLane> B) { seg_bbox_body(B.a[blockIdx.z].f); }


// grid (chunks, segments): keys / vals in the compact order (segment after segment)
__device__ __forceinline__ void seg_keys_body(SegFilter f, unsigned* __restrict__ keys, int* __restrict__ vals) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int sgm = blockIdx.y;
  if (sgm >= seg_count(f)) return;
  const SegDesc d = f.seg[f.seg0 + sgm];
  const int n = *d.n_in;
  if (n <= 0) return;
  const int off = f.off[sgm];
  float mn[3], mx[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) { mn[a] = ord2f(f.bbox[6 * sgm + a]); mx[a] = ord2f(f.bbox[6 * sgm + 3 + a]); }
  const float inv = 1.0f / d.leaf;
  long long dxyz[3]; int min_b[3], div_b[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    dxyz[a] = (long long)((mx[a] - mn[a]) * inv) + 1;
    min_b[a] = (int)floorf(mn[a] * inv);
    div_b[a] = (int)floorf(mx[a] * inv) - min_b[a] + 1;
  }
  const unsigned long long cells = (unsigned long long)div_b[0] * (unsigned long long)div_b[1] * (unsigned long long)div_b[2];
  const bool pcl_overflow = dxyz[0] * dxyz[1] * dxyz[2] > (long long)INT_MAX;   // PCL: "leaf size is too small", input returned unchanged
  // cannot be encoded: flagged, points kept as they are.  At 32 bits the key is PCL's own int index and wraps as PCL's does.
  const bool key_overflow = !pcl_overflow && f.idx_bits < 32 && cells > (1ull << f.idx_bits);
  const bool pass = pcl_overflow || key_overflow;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    f.pass[sgm] = pass;
    if (key_overflow) atomicOr(f.err, 1);
  }
  const unsigned hi_bits = (unsigned)((unsigned long long)sgm << f.idx_bits);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned idx;
    if (pass) idx = (unsigned)i;
    else {
      const Pt4 p = d.src[i];
      const int i0 = (int)(floorf(p.x * inv) - (float)min_b[0]);
      const int i1 = (int)(floorf(p.y * inv) - (float)min_b[1]);
      const int i2 = (int)(floorf(p.z * inv) - (float)min_b[2]);
      idx = (unsigned)(i0 + i1 * div_b[0] + i2 * div_b[0] * div_b[1]);
    }
    keys[off + i] = hi_bits | idx;
    vals[off + i] = off + i;
  }
}
__global__ void __launch_bounds__(256) k_seg_keys(const __grid_constant__ Batch<VoxLane> B) {
  const VoxLane& a = B.a[blockIdx.z];
  seg_keys_body(a.f, a.keys[0], a.vals[0]);
}


// heads before the first sorted slot of every segment (grid: segments + 1 CTAs of one warp; CTA s ranks slot off[s])
__device__ __forceinline__ int seg_head_rank(const unsigned* __restrict__ keys, const int* __restrict__ block_offsets, int pos, int total) {
  const int lane = threadIdx.x & 31;
  if (total <= 0) return 0;
  const int p = min(pos, total);
  // heads in [block start, p): for p == total the block is the last one (all of its heads count)
  const int b = p >= total ? (total - 1) / VCH : p / VCH;
  int cnt = 0;
  for (int i = b * VCH + lane; i < p; i += 32) cnt += (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
#pragma unroll
  for (int dd = 16; dd > 0; dd >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, dd);
  return block_offsets[b] + cnt;
}
__device__ __forceinline__ void seg_rank0_body(SegFilter f, const unsigned* __restrict__ keys, const int* __restrict__ block_offsets) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int S = seg_count(f), total = *f.total;
  const int sgm = blockIdx.x;
  if (sgm > S) return;
  const int r0 = seg_head_rank(keys, block_offsets, sgm == S ? total : f.off[sgm], total);
  if (threadIdx.x == 0) f.rank0[sgm] = r0;
  if (sgm < S) {   // the filtered size of this segment needs the rank of the next boundary too
    const int r1 = seg_head_rank(keys, block_offsets, sgm + 1 == S ? total : f.off[sgm + 1], total);
    if (threadIdx.x == 0) *f.seg[f.seg0 + sgm].n_out = r1 - r0;
  }
}
__global__ void __launch_bounds__(32) k_seg_rank0(const __grid_constant__ Batch<VoxLane> B, int cur) {
  const VoxLane& a = B.a[blockIdx.z];
  seg_rank0_body(a.f, a.keys[cur], a.block_heads);
}


// every head sums its run in sorted order (float, like pcl::CentroidPoint); output slot = off[segment] + rank inside the segment.
// The CTAs stride over the blocks of VCH sorted keys (the grid is sized by a host bound, the live total is on the device).
__device__ __forceinline__ void seg_emit_body(SegFilter f, const unsigned* __restrict__ keys, const int* __restrict__ vals,
                                                 const int* __restrict__ block_offsets, Pt4* __restrict__ tmp) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int n = *f.total;
  __shared__ int s_w[VT / 32];
  __shared__ Pt4 s_pts[VCH];        // the block's points in sorted order: the runs are summed from shared memory, the gather
  __shared__ unsigned s_keys[VCH];  // through vals[] is issued once, all loads in flight
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int blk = blockIdx.x; blk * VCH < n; blk += gridDim.x) {
    const int b0 = blk * VCH;
#pragma unroll
    for (int k = 0; k < VIT; ++k) {
      const int i = b0 + k * VT + tid;
      if (i < n) {
        const unsigned key = keys[i];
        const int sgm = seg_of(key, f.idx_bits);
        s_keys[k * VT + tid] = key;
        s_pts[k * VT + tid] = f.seg[f.seg0 + sgm].src[vals[i] - f.off[sgm]];
      }
    }
    __syncthreads();
    const int base = b0 + tid * VIT;
    int heads = 0;
    bool is_head[VIT];
#pragma unroll
    for (int k = 0; k < VIT; ++k) {
      const int i = base + k;
      is_head[k] = i < n && (i == 0 || keys[i] != keys[i - 1]);
      heads += is_head[k] ? 1 : 0;
    }
    int incl = heads;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
    if (lane == 31) s_w[w] = incl;
    __syncthreads();
    int wbase = 0;
    for (int v = 0; v < w; ++v) wbase += s_w[v];
    int rank = block_offsets[blk] + wbase + incl - heads;
    const int bend = min(n, b0 + VCH);
#pragma unroll
    for (int k = 0; k < VIT; ++k) {
      if (!is_head[k]) continue;
      const int i = base + k;
      const unsigned key = s_keys[i - b0];
      const int sgm = seg_of(key, f.idx_bits);
      const int off = f.off[sgm];
      float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
      int cnt = 0;
      int j = i;
      for (; j < bend && s_keys[j - b0] == key; ++j) {   // float accumulation in sorted order (pcl::CentroidPoint)
        const Pt4 p = s_pts[j - b0];
        sx += p.x; sy += p.y; sz += p.z; si += p.i;
        ++cnt;
      }
      if (j == bend) {   // the run continues in the next block(s): finish it from global memory
        const Pt4* __restrict__ src = f.seg[f.seg0 + sgm].src;
        for (; j < n && keys[j] == key; ++j) {
          const Pt4 p = src[vals[j] - off];
          sx += p.x; sy += p.y; sz += p.z; si += p.i;
          ++cnt;
        }
      }
      const float nf = (float)cnt;
      Pt4 o; o.x = sx / nf; o.y = sy / nf; o.z = sz / nf; o.i = si / nf;
      tmp[off + (rank - f.rank0[sgm])] = o;
      ++rank;
    }
    __syncthreads();   // s_w, s_pts and s_keys are refilled for the next block
  }
}
__global__ void __launch_bounds__(VT) k_seg_emit(const __grid_constant__ Batch<VoxLane> B, int cur) {
  const VoxLane& a = B.a[blockIdx.z];
  seg_emit_body(a.f, a.keys[cur], a.vals[cur], a.block_heads, a.tmp);
}


// grid (chunks, segments): filtered points back to their destination (which may be the source slab itself).  A pass-through
// segment is copied from its source, not from its one-point "centroids": (0.f + x) / 1.f would turn -0.f into +0.f.
__device__ __forceinline__ void seg_writeback_body(SegFilter f, const Pt4* __restrict__ tmp) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int sgm = blockIdx.y;
  if (sgm >= seg_count(f)) return;
  const SegDesc d = f.seg[f.seg0 + sgm];
  const int m = f.rank0[sgm + 1] - f.rank0[sgm];   // a pass-through segment has one key per point: m is its size
  const bool pass = f.pass[sgm];                   // not set for an empty segment, which has m = 0
  if (pass && d.dst == d.src) return;
  const Pt4* __restrict__ from = pass ? d.src : tmp + f.off[sgm];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) d.dst[i] = from[i];
}
__global__ void __launch_bounds__(256) k_seg_writeback(const __grid_constant__ Batch<VoxLane> B) {
  const VoxLane& a = B.a[blockIdx.z];
  seg_writeback_body(a.f, a.tmp);
}


}  // namespace aloam

using namespace aloam;

// segmented filter over up to S_upper segments in each of nb lanes (filter f[l] on buffers *b[l]); every launch covers all lanes,
// lane l in blockIdx.z.  n_upper / per_seg_upper are host bounds per lane for grid sizing (total points, points of one segment).
// The caller guarantees that a lane's live total never exceeds its b[l]->cap: nothing here clamps it.  A 32-bit key holds
// f.idx_bits index bits and the segment number: when S_upper segments do not fit beside the index, the segments are processed
// in windows of 2^(32 - idx_bits) (idx_bits = 32: one segment, 32 key bits); idx_bits is the same in every lane.
void vox_seg_filter(aloam_ctx* c, int nb, const SegFilter* f_in, SegBuffers* const* b, int S_upper, int n_upper, int per_seg_upper) {
  const int nblk = std::max(1, (n_upper + VCH - 1) / VCH);
  const int grid_blk = std::min(nblk, std::max(1, 8 * c->sms / nb));   // k_vox_heads / k_seg_emit stride over the blocks: one resident wave at most
  const int chunks = std::max(1, std::min((per_seg_upper + 255) / 256, S_upper > 8 ? 8 : 64));   // grid-stride inside a segment
  const int idx_bits = f_in[0].idx_bits;
  const int win = (int)std::min<long long>(1ll << std::max(0, 32 - idx_bits), ALOAM_MAX_SEGS);
  for (int s0 = 0; s0 < S_upper; s0 += win) {
    const int seg_cap = std::min(win, S_upper - s0);
    Batch<VoxLane> B = {};
    for (int l = 0; l < nb; ++l) {
      SegFilter f = f_in[l];
      f.seg0 = s0; f.seg_cap = seg_cap;
      const SegBuffers& bl = *b[l];
      B.a[l] = VoxLane{f, {bl.keys[0], bl.keys[1]}, {bl.vals[0], bl.vals[1]}, bl.hist, bl.block_heads, bl.heads_total, bl.tmp};
    }
    int seg_bits = 0; while ((1 << seg_bits) < seg_cap) ++seg_bits;
    const int bits = idx_bits + seg_bits;
    launch_ex(c, KID_VOXEL, k_seg_prep, dim3(1, 1, nb), dim3(256), 0, 1, true, B);
    launch_ex(c, KID_VOXEL, k_seg_bbox, dim3(chunks, seg_cap, nb), dim3(256), 0, 1, true, B);
    launch_ex(c, KID_VOXEL, k_seg_keys, dim3(chunks, seg_cap, nb), dim3(256), 0, 1, true, B);
    // the radix passes: one cooperative launch (all CTAs co-resident, at most one per SM over all lanes)
    {
      prof_begin(c, KID_VOXEL);
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(std::min(nblk, std::max(1, b[0]->coop_grid / nb)), 1, nb); cfg.blockDim = dim3(VT); cfg.dynamicSmemBytes = 0; cfg.stream = c->stream;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      cudaLaunchKernelEx(&cfg, k_radix_sort_all, B, bits);
      prof_end(c);
    }
    const int cur = ((bits + 7) / 8) & 1;
    launch_ex(c, KID_VOXEL, k_vox_heads, dim3(grid_blk, 1, nb), dim3(VT), 0, 1, true, B, cur);
    launch_ex(c, KID_VOXEL, k_vox_blockscan, dim3(1, 1, nb), dim3(1024), 0, 1, true, B);
    launch_ex(c, KID_VOXEL, k_seg_rank0, dim3(seg_cap + 1, 1, nb), dim3(32), 0, 1, true, B, cur);
    launch_ex(c, KID_VOXEL, k_seg_emit, dim3(grid_blk, 1, nb), dim3(VT), 0, 1, true, B, cur);
    launch_ex(c, KID_VOXEL, k_seg_writeback, dim3(chunks, seg_cap, nb), dim3(256), 0, 1, true, B);
  }
}

// a stable LSD sort of the *n_dev (<= n_upper) keys k0 / values v0 by their low `bits` bits, one cooperative launch; the result is
// in (k0, v0) when bits / 8 is even, else in (k1, v1).  hist holds 256 ints per tile of VCH keys.  Kernel id kid.
int vox_radix_sort(aloam_ctx* c, int kid, unsigned* k0, int* v0, unsigned* k1, int* v1, const int* n_dev, int n_upper, int bits, int* hist) {
  int per_sm = 0;
  CUDA_CHECK_RET(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_radix_sort_flat, VT, 0));
  const int tiles = std::max(1, (n_upper + VCH - 1) / VCH);
  prof_begin(c, kid);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(std::min(tiles, std::max(1, per_sm * c->sms))); cfg.blockDim = dim3(VT); cfg.dynamicSmemBytes = 0; cfg.stream = c->stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, k_radix_sort_flat, k0, v0, k1, v1, n_dev, bits, hist);
  prof_end(c);
  CUDA_CHECK_RET(e);
  return ALOAM_OK;
}
size_t vox_radix_hist_ints(int n) { return (size_t)std::max(1, (n + VCH - 1) / VCH) * 256; }

int vox_seg_alloc(aloam_ctx* c, BufGroup& g, SegBuffers& b, size_t cap) {
  const size_t nb = (cap + VCH - 1) / VCH + 1;
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_radix_sort_all, VT, 0);
  b.cap = cap;
  b.coop_grid = std::max(1, std::min(c->sms, per_sm * c->sms));
  if (!g.dev(&b.segs, ALOAM_MAX_SEGS) || !g.dev(&b.n_seg, 1) || !g.dev(&b.off, ALOAM_MAX_SEGS + 8) || !g.dev(&b.rank0, ALOAM_MAX_SEGS + 8) ||
      !g.dev(&b.bbox, ALOAM_MAX_SEGS * 6) || !g.dev(&b.total, 1) || !g.dev(&b.pass, ALOAM_MAX_SEGS) || !g.dev(&b.keys[0], cap) ||
      !g.dev(&b.keys[1], cap) || !g.dev(&b.vals[0], cap) || !g.dev(&b.vals[1], cap) || !g.dev(&b.hist, nb * 256) ||
      !g.dev(&b.block_heads, nb) || !g.dev(&b.heads_total, 1) || !g.dev(&b.tmp, cap))
    return ALOAM_ERR_CUDA;
  return ALOAM_OK;
}

// the general entry point: the cloud is the one segment of a segmented filter the context owns for it (not the mapper's)
extern "C" int aloam_voxel_filter(aloam_ctx* c, aloam_cloud_view in, float leaf, aloam_cloud_view* out) {
  if (!c || !out || !(leaf > 0.f)) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(in); if (rc) return rc;
  if (in.n > c->max_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  // the result has its OWN pinned buffer: a caller may pass a view returned by aloam_extract_features (h_out[*]) straight
  // back in, so the output must not alias any other ctx-owned view
  if (!c->h_vox_out) CUDA_CHECK_RET(halloc(c, &c->h_vox_out, (size_t)c->max_points));
  out->data = reinterpret_cast<const float*>(c->h_vox_out); out->n = 0; out->stride_floats = 4;
  if (in.n == 0) return ALOAM_OK;
  if (!c->d_seg_io) {   // first use: the filter and its io words, one group published complete
    BufGroup g;
    SegBuffers b;
    int* io;
    if (!g.dev(&io, 3) || vox_seg_alloc(c, g, b, (size_t)c->max_points) != ALOAM_OK) return ALOAM_ERR_CUDA;
    own(c, std::move(g));
    c->vox_seg = b;
    c->d_seg_io = io;
  }
  Pt4* d_in = c->d_query;        // staging buffers that already exist in the context
  Pt4* d_out = c->lanes[0].d_full[0];
  rc = upload_cloud(c, in, d_in, c->max_points); if (rc) return rc;
  SegBuffers& b = c->vox_seg;
  int* io = c->d_seg_io;     // cloud size, filtered size, error word
  PinnedScratch* p = c->pin;
  p->vox_seg = SegDesc{d_in, io, leaf, d_out, io + 1};
  p->vox_nseg = 1;
  p->vox_io[0] = in.n; p->vox_io[1] = 0; p->vox_io[2] = 0;
  CUDA_CHECK_RET(cudaMemcpyAsync(b.segs, &p->vox_seg, sizeof(SegDesc), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(b.n_seg, &p->vox_nseg, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(io, p->vox_io, sizeof(p->vox_io), cudaMemcpyHostToDevice, c->stream));
  // 32 index bits: the key is PCL's int index itself, so every cloud PCL filters is filtered here and the error word stays 0
  const SegFilter f = seg_filter(b, 32, io + 2);
  SegBuffers* bp = &b;
  vox_seg_filter(c, 1, &f, &bp, 1, in.n, in.n);
  CUDA_CHECK_RET(cudaMemcpyAsync(&p->vox_out_n, io + 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  const int m = p->vox_out_n;
  if (m > 0) {
    CUDA_CHECK_RET(cudaMemcpyAsync(c->h_vox_out, d_out, (size_t)m * 16, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  }
  prof_collect(c);
  out->n = m;
  return ALOAM_OK;
}
