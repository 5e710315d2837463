// Scan-to-map association on the GPU -- replaces laserMapping.cpp:154-163 (pointAssociateToMap), :558-559 (the two
// kd-tree builds over the gathered submap), :577-622 (corner: 5-NN, covariance, eigen line test, LidarEdgeFactor)
// and :643-687 (surf: 5-NN, plane fit, LidarPlaneNormFactor).
//
// K0  map index = hash grid with cell edge 1 m * (1 + 1e-5): the reference only uses a neighbourhood whose 5th
//     member is closer than 1 m (`pointSearchSqDis[4] < 1.0`, :584,652), so every neighbour that can matter lies in
//     the 3 x 3 x 3 cells around the query and one probe round (27 lanes) replaces the O(M log M) kd-tree build +
//     descent.  The table is sized to the cloud actually indexed (next power of two above 1.25 n, not to the context
//     capacity: the round-1 table was cleared and scanned at capacity, 5x the algorithmic traffic) and one slot is ONE
//     16-byte word {cell key (64 bit), count, end}: a probe is a single LDG.128.  Build = clear / insert (atomicCAS on
//     the key, atomicAdd on the count) / alloc (block scan, one cursor atomic per CTA) / fill (re-probe, atomicAdd on
//     the slot's running end) -- no per-point scratch arrays.  Order inside a cell depends on atomic timing;
//     selection is on (distance, original index) so results do not.
// K5  k_map_knn5: one warp per stack point: probe 27 cells, flatten their points with a warp scan, every lane keeps its
//     own sorted top-5, five REDUX arg-min rounds merge them into the exact 5-NN in ascending (distance, index) order;
//     lanes 0..4 fetch the five winners and store them (80 B per query).
// K6  k_map_fit: one THREAD per stack point fits the line (3x3 symmetric eigen, Jacobi) or the plane (5x3 least
//     squares, Householder) in double precision exactly as the oracle does and writes the residual block the LM kernel
//     consumes.  (Round 1 ran the fit on lane 0 of the search warp: 31 idle lanes for the longest serial section.)
// Every size is read from device memory (GridDyn / counts), so the same kernels serve the host-driven API
// (aloam_map_upload / aloam_mapping_register) and the device-resident mapping loop (cubemap.cu) without a host sync.
// Multi-GPU: a rank only fits the queries whose cell it owns (slabs of 8 cells along x, round-robin over ranks); its
//     shard of the map holds those slabs plus a one-cell halo, so its 27-cell neighbourhoods are complete.
#include <cfloat>
#include <climits>
#include <nccl.h>
#include "ctx.h"
#include "grid.cuh"

namespace aloam {

namespace {
constexpr int kSlab = 8;  // cells per ownership slab (x direction)

// floor division and a non-negative remainder, as shard.py's owner_of_cell: a cell left of x = -2^20 m still has an owner
__device__ __forceinline__ int owner_of(int cx, int count) {
  const int v = cx + (1 << 20);
  const int slab = (v < 0 ? v - (kSlab - 1) : v) / kSlab;
  const int r = slab % count;
  return r < 0 ? r + count : r;
}
__device__ __forceinline__ unsigned table_mask_for(int n) {   // next power of two >= 1.25 n (>= 1024), minus one
  unsigned want = (unsigned)n + ((unsigned)n >> 2);
  unsigned m = 1024;
  while (m < want) m <<= 1;
  return m - 1;
}
}  // namespace

unsigned grid_mask_for(int n, unsigned cap_slots) {
  unsigned want = (unsigned)n + ((unsigned)n >> 2);
  unsigned m = 1024;
  while (m < want && m < cap_slots) m <<= 1;
  return m - 1;
}

// device-resident sizes -> GridDyn (the mapping loop gathers the submap on the device; its size never visits the host)
__device__ __forceinline__ void grid_setup_body(GridTable a, const int* __restrict__ na, GridTable b, const int* __restrict__ nb) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    a.dyn->n = *na; a.dyn->mask = min(table_mask_for(*na), a.cap_slots - 1); a.dyn->cursor = 0; a.dyn->owned = 0;
    b.dyn->n = *nb; b.dyn->mask = min(table_mask_for(*nb), b.cap_slots - 1); b.dyn->cursor = 0; b.dyn->owned = 0;
  }
}
// grid (1, 1, lanes)
__global__ void k_grid_setup(const __grid_constant__ Batch<GridArgs> B) { const GridArgs& g = B.a[blockIdx.z]; grid_setup_body(g.a, g.na, g.b, g.nb); }


__device__ __forceinline__ void grid_clear_body(GridTable a, GridTable b) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gstride = gridDim.x * blockDim.x;
  const uint4 empty = make_uint4(~0u, ~0u, 0u, 0u);
  const int ma = (int)a.dyn->mask, mb = (int)b.dyn->mask;
  for (int i = gtid; i <= ma; i += gstride) a.slots[i] = empty;
  for (int i = gtid; i <= mb; i += gstride) b.slots[i] = empty;
}
// grid (CTAs, 1, lanes)
__global__ void k_grid_clear(const __grid_constant__ Batch<GridArgs> B) { const GridArgs& g = B.a[blockIdx.z]; grid_clear_body(g.a, g.b); }


// blockIdx.y selects the cloud (0 = a, 1 = b).  (Grouping the lanes of a cell with __match_any so that one lane claims the slot for
// the group was tried here and was slower -- the vote costs more than the atomics it saves; the fill below does profit from
// it.)
__device__ __forceinline__ void grid_insert_body(GridTable a, const Pt4* __restrict__ pa, GridTable b, const Pt4* __restrict__ pb, int shard_rank,
                              int shard_count) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const GridTable& g = blockIdx.y == 0 ? a : b;
  const Pt4* __restrict__ pts = blockIdx.y == 0 ? pa : pb;
  const int n = g.dyn->n;
  const unsigned mask = g.dyn->mask;
  int owned = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const Pt4 p = pts[i];
    const int cx = cell_of(p.x, g.inv_cs);
    const unsigned long long key = cell_key(cx, cell_of(p.y, g.inv_cs), cell_of(p.z, g.inv_cs));
    unsigned h = hash_key(key) & mask;
    for (;;) {
      const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(&g.slots[h]), kEmpty, key);
      if (prev == kEmpty || prev == key) break;
      h = (h + 1) & mask;
    }
    atomicAdd(reinterpret_cast<int*>(&g.slots[h]) + 2, 1);
    if (shard_count > 1 && owner_of(cx, shard_count) == shard_rank) ++owned;
  }
  if (shard_count > 1) {   // points in cells this rank owns (the halo excluded): the global map size is their sum over ranks
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) owned += __shfl_xor_sync(0xffffffffu, owned, d);
    if ((threadIdx.x & 31) == 0 && owned) atomicAdd(&g.dyn->owned, owned);
  }
}
// grid (CTAs, 2 clouds, lanes)
__global__ void k_grid_insert(const __grid_constant__ Batch<GridArgs> B, int shard_rank, int shard_count) {
  const GridArgs& g = B.a[blockIdx.z];
  grid_insert_body(g.a, g.pa, g.b, g.pb, shard_rank, shard_count);
}


// per-cell storage: block-wide exclusive scan of the counts, ONE atomicAdd per CTA and table on the cursor (a per-slot
// atomicAdd serialises ~500k updates of a single address for a 1M-point map).  Writes the cell's START
// into the `end` word; k_grid_fill advances it to the end.
__device__ __forceinline__ void grid_alloc_body(GridTable a, GridTable b) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  __shared__ int s_w[2][8];
  __shared__ int s_base[2];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int ma = (int)a.dyn->mask, mb = (int)b.dyn->mask;
  const int tiles = (max(ma, mb) + 256) / 256;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int i = tile * 256 + threadIdx.x;
    int c[2], incl[2];
    c[0] = i <= ma ? (int)a.slots[i].z : 0;
    c[1] = i <= mb ? (int)b.slots[i].z : 0;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      int v = c[t];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += u; }
      incl[t] = v;
      if (lane == 31) s_w[t][w] = v;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
      int tot = 0;
      for (int k = 0; k < 8; ++k) { const int x = s_w[threadIdx.x][k]; s_w[threadIdx.x][k] = tot; tot += x; }
      s_base[threadIdx.x] = tot > 0 ? atomicAdd(threadIdx.x == 0 ? &a.dyn->cursor : &b.dyn->cursor, tot) : 0;
    }
    __syncthreads();
    if (i <= ma && c[0] > 0) reinterpret_cast<int*>(&a.slots[i])[3] = s_base[0] + s_w[0][w] + incl[0] - c[0];
    if (i <= mb && c[1] > 0) reinterpret_cast<int*>(&b.slots[i])[3] = s_base[1] + s_w[1][w] + incl[1] - c[1];
    __syncthreads();
  }
}
// grid (CTAs, 1, lanes)
__global__ void __launch_bounds__(256) k_grid_alloc(const __grid_constant__ Batch<GridArgs> B) { const GridArgs& g = B.a[blockIdx.z]; grid_alloc_body(g.a, g.b); }


__device__ __forceinline__ void grid_fill_body(GridTable a, const Pt4* __restrict__ pa, GridTable b, const Pt4* __restrict__ pb) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const GridTable& g = blockIdx.y == 0 ? a : b;
  const Pt4* __restrict__ pts = blockIdx.y == 0 ? pa : pb;
  const int n = g.dyn->n;
  const unsigned mask = g.dyn->mask;
  const unsigned lane = lane_id();
  const int stride = gridDim.x * blockDim.x;
  for (int i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31); i0 < n; i0 += stride) {
    const int i = i0 + (int)lane;
    unsigned long long key = kEmpty;
    Pt4 p = {0.f, 0.f, 0.f, 0.f};
    if (i < n) {
      p = pts[i];
      key = cell_key(cell_of(p.x, g.inv_cs), cell_of(p.y, g.inv_cs), cell_of(p.z, g.inv_cs));
    }
    const unsigned grp = __match_any_sync(0xffffffffu, key);
    const int leader = __ffs(grp) - 1;
    int base = 0;
    if (i < n && (int)lane == leader) {   // one probe and one atomic per group of lanes in the same cell
      unsigned h = hash_key(key) & mask;
      while (*reinterpret_cast<const volatile unsigned long long*>(&g.slots[h]) != key) h = (h + 1) & mask;   // inserted by k_grid_insert
      base = atomicAdd(reinterpret_cast<int*>(&g.slots[h]) + 3, __popc(grp));
    }
    base = __shfl_sync(0xffffffffu, base, leader);
    if (i < n) g.gpts[base + __popc(grp & ((1u << lane) - 1u))] = make_float4(p.x, p.y, p.z, __int_as_float(i));
  }
}
// grid (CTAs, 2 clouds, lanes)
__global__ void k_grid_fill(const __grid_constant__ Batch<GridArgs> B) { const GridArgs& g = B.a[blockIdx.z]; grid_fill_body(g.a, g.pa, g.b, g.pb); }


// ---- device-side shard split (SURVEY.md 8e): keeps the points of a cloud that fall in this rank's x-slabs or within one
// cell of them (the halo), in their original order -- a stable stream compaction in three launches (per-block counts, scan of
// the block counts, scatter).  `base` (device) is the number of points already kept by earlier chunks of the same cloud.
__device__ __forceinline__ bool in_shard(float x, float inv_cs, int rank, int world) {
  const int cx = cell_of(x, inv_cs);
  return owner_of(cx, world) == rank || owner_of(cx - 1, world) == rank || owner_of(cx + 1, world) == rank;
}
// (n_ptr != nullptr: the number of points lives on the device -- the submap gathered by the mapper -- and n is only the launch bound)
__global__ void __launch_bounds__(256) k_shard_count(const float* __restrict__ pts, int stride, int n, const int* __restrict__ n_ptr, float inv_cs, int rank, int world,
                                                     int* __restrict__ block_cnt) {
  if (n_ptr) n = min(n, *n_ptr);
  const int i = blockIdx.x * 256 + threadIdx.x;
  const bool keep = i < n && in_shard(pts[(size_t)i * stride], inv_cs, rank, world);
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_cnt[blockIdx.x] = c;
}
// *base_total ends clamped to cap: the points k_shard_scatter cannot store (it flags them) never reach the index build
__global__ void __launch_bounds__(1024) k_shard_scan(int* __restrict__ block_cnt, int nblocks, int* __restrict__ base_total, int cap) {
  __shared__ int s_w[32];
  __shared__ int s_carry;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  if (t == 0) s_carry = *base_total;
  __syncthreads();
  for (int b0 = 0; b0 < nblocks; b0 += 1024) {
    const int b = b0 + t;
    const int v = b < nblocks ? block_cnt[b] : 0;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
    if (lane == 31) s_w[w] = incl;
    __syncthreads();
    int wb = 0;
    for (int k = 0; k < w; ++k) wb += s_w[k];
    const int carry = s_carry;
    if (b < nblocks) block_cnt[b] = carry + wb + incl - v;
    __syncthreads();
    if (t == 1023) s_carry = carry + wb + incl;
    __syncthreads();
  }
  if (t == 0) *base_total = min(s_carry, cap);
}
__global__ void __launch_bounds__(256) k_shard_scatter(const float* __restrict__ pts, int stride, int n, const int* __restrict__ n_ptr, float inv_cs, int rank, int world,
                                                       const int* __restrict__ block_off, Pt4* __restrict__ out, int cap, int* __restrict__ err) {
  __shared__ int s_w[8];
  if (n_ptr) n = min(n, *n_ptr);
  const int i = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  Pt4 p = {0.f, 0.f, 0.f, 0.f};
  bool keep = false;
  if (i < n) {
    const float* q = pts + (size_t)i * stride;
    p.x = q[0]; p.y = q[1]; p.z = q[2]; p.i = q[3];
    keep = in_shard(p.x, inv_cs, rank, world);
  }
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) s_w[w] = __popc(bal);
  __syncthreads();
  int wb = 0;
  for (int k = 0; k < w; ++k) wb += s_w[k];
  if (keep) {
    const int pos = block_off[blockIdx.x] + wb + __popc(bal & ((1u << lane) - 1u));
    if (pos < cap) out[pos] = p; else atomicOr(err, 1);
  }
}

namespace {

// per-lane sorted list of the K best (distance, original index) with the point's slot in gpts as payload
template <int K>
struct TopK {
  float d[K]; int i[K]; int p[K];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < K; ++k) { d[k] = FLT_MAX; i[k] = INT_MAX; p[k] = 0; }
  }
  __device__ __forceinline__ void push(float dd, int ii, int pp) {   // keep ascending (d, i)
    if (!(dd < d[K - 1] || (dd == d[K - 1] && ii < i[K - 1]))) return;
    d[K - 1] = dd; i[K - 1] = ii; p[K - 1] = pp;
#pragma unroll
    for (int k = K - 1; k > 0; --k) {
      const bool sw = d[k] < d[k - 1] || (d[k] == d[k - 1] && i[k] < i[k - 1]);
      if (sw) {
        float td = d[k]; d[k] = d[k - 1]; d[k - 1] = td;
        int ti = i[k]; i[k] = i[k - 1]; i[k - 1] = ti;
        int tp = p[k]; p[k] = p[k - 1]; p[k - 1] = tp;
      }
    }
  }
  __device__ __forceinline__ void pop() {
#pragma unroll
    for (int k = 0; k < K - 1; ++k) { d[k] = d[k + 1]; i[k] = i[k + 1]; p[k] = p[k + 1]; }
    d[K - 1] = FLT_MAX; i[K - 1] = INT_MAX;
  }
};

// all points of the 27 cells around q go through f(x, y, z, index, slot), each exactly once, on some lane
template <typename F>
__device__ __forceinline__ void visit_block27(const GridTable& g, unsigned mask, float qx, float qy, float qz, F&& f) {
  const int lane = (int)lane_id();
  const int cx = cell_of(qx, g.inv_cs), cy = cell_of(qy, g.inv_cs), cz = cell_of(qz, g.inv_cs);
  int start = 0, cnt = 0;
  if (lane < 27) {
    const int dz = lane / 9 - 1, dy = (lane % 9) / 3 - 1, dx = lane % 3 - 1;
    const unsigned long long key = cell_key(cx + dx, cy + dy, cz + dz);
    unsigned h = hash_key(key) & mask;
    for (;;) {
      const uint4 s = __ldg(g.slots + h);   // one 16-byte probe: key, count, end
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
    if (e < total) {
      const int slot = c_start + (e - (c_incl - c_cnt));
      const float4 p = __ldg(g.gpts + slot);
      f(p.x, p.y, p.z, __float_as_int(p.w), slot);
    }
  }
}

// merges the lanes' sorted lists: out[k] = k-th smallest (d, i) of the warp and its gpts slot, warp-uniform ; returns how many exist
template <int K>
__device__ __forceinline__ int warp_merge_topk(TopK<K>& t, float* out_d, int* out_i, int* out_p) {
  int found = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    float d = t.d[0]; int i = t.i[0];
    warp_argmin(d, i);
    out_d[k] = d; out_i[k] = i; out_p[k] = 0;
    if (i != INT_MAX && d != FLT_MAX) {
      ++found;
      const bool mine = t.i[0] == i && t.d[0] == d;
      const unsigned own = __ballot_sync(0xffffffffu, mine);
      out_p[k] = __shfl_sync(0xffffffffu, t.p[0], __ffs(own) - 1);
      if (mine) t.pop();
    }
  }
  return found;
}

// 3x3 symmetric eigen-decomposition, cyclic Jacobi (same rotations as the oracle's eig3_sym): ascending eigenvalues,
// vmax = unit eigenvector of the largest one.  Fully unrolled: every array index is a compile-time constant, so the
// matrices live in registers.
__device__ __forceinline__ void eig3_sym(const double (&Ain)[9], double (&evals)[3], double (&vmax)[3]) {
  double A[9], V[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) { A[i] = Ain[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 64; ++sweep) {
    const double off = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    const double dsum = A[0] * A[0] + A[4] * A[4] + A[8] * A[8];
    if (off <= 1e-32 * dsum || off == 0.0) break;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        const double apq = A[3 * p + q];
        if (apq != 0.0) {
          const double theta = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
          const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
          for (int k = 0; k < 3; ++k) { const double akp = A[3 * k + p], akq = A[3 * k + q]; A[3 * k + p] = c * akp - s * akq; A[3 * k + q] = s * akp + c * akq; }
#pragma unroll
          for (int k = 0; k < 3; ++k) { const double apk = A[3 * p + k], aqk = A[3 * q + k]; A[3 * p + k] = c * apk - s * aqk; A[3 * q + k] = s * apk + c * aqk; }
#pragma unroll
          for (int k = 0; k < 3; ++k) { const double vkp = V[3 * k + p], vkq = V[3 * k + q]; V[3 * k + p] = c * vkp - s * vkq; V[3 * k + q] = s * vkp + c * vkq; }
        }
      }
    }
  }
  // sort the three (eigenvalue, eigenvector) pairs ascending with static compare-exchanges
  double e0 = A[0], e1 = A[4], e2 = A[8];
  double v0[3] = {V[0], V[3], V[6]}, v1[3] = {V[1], V[4], V[7]}, v2[3] = {V[2], V[5], V[8]};
#define ALOAM_CSWAP(ea, va, eb, vb) if (eb < ea) { double te = ea; ea = eb; eb = te; for (int k = 0; k < 3; ++k) { double tv = va[k]; va[k] = vb[k]; vb[k] = tv; } }
  ALOAM_CSWAP(e0, v0, e1, v1)
  ALOAM_CSWAP(e1, v1, e2, v2)
  ALOAM_CSWAP(e0, v0, e1, v1)
#undef ALOAM_CSWAP
  evals[0] = e0; evals[1] = e1; evals[2] = e2;
#pragma unroll
  for (int k = 0; k < 3; ++k) vmax[k] = v2[k];
}

// least squares A n = b (5x3) with Eigen's colPivHouseholderQr().solve semantics, fully unrolled (registers): Householder
// QR pivoting on the remaining column of largest norm (first index on ties); rank = number of |R_kk| > 3 eps max|R_kk|;
// back-substitution over the leading rank x rank block, the other unknowns 0.  A collinear or duplicated neighbourhood
// (rank 1 or 2) therefore gives the same finite basic solution as Eigen instead of a 0/0 normal.  Every operation is in a
// fixed order and this file is built -fmad=false, so a CPU restatement with the same order agrees bit for bit.
__device__ __forceinline__ void lsq_5x3(const double (&Ain)[15], const double (&bin)[5], double (&n)[3]) {
  double A[15], b[5];
  int perm[3] = {0, 1, 2};
#pragma unroll
  for (int i = 0; i < 15; ++i) A[i] = Ain[i];
#pragma unroll
  for (int i = 0; i < 5; ++i) b[i] = bin[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int best = k;
    double norm2 = -1;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (j >= k) {
        double s = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) if (i >= k) s += A[3 * i + j] * A[3 * i + j];
        if (s > norm2) { norm2 = s; best = j; }
      }
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {   // swap columns k and best (whole columns, as the oracle) with static indices
      if (j > k && best == j) {
#pragma unroll
        for (int i = 0; i < 5; ++i) { const double t = A[3 * i + k]; A[3 * i + k] = A[3 * i + j]; A[3 * i + j] = t; }
        const int tp = perm[k]; perm[k] = perm[j]; perm[j] = tp;
      }
    }
    const double nrm = sqrt(norm2);
    const double akk = A[3 * k + k];
    const double alpha = akk > 0 ? -nrm : nrm;
    const double v0 = akk - alpha;
    const double vn2 = norm2 - akk * akk + v0 * v0;
    A[3 * k + k] = v0;
    if (vn2 > 0) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        if (j > k) {
          double s = 0;
#pragma unroll
          for (int i = 0; i < 5; ++i) if (i >= k) s += A[3 * i + k] * A[3 * i + j];
          s = 2.0 * s / vn2;
#pragma unroll
          for (int i = 0; i < 5; ++i) if (i >= k) A[3 * i + j] -= s * A[3 * i + k];
        }
      }
      double s = 0;
#pragma unroll
      for (int i = 0; i < 5; ++i) if (i >= k) s += A[3 * i + k] * b[i];
      s = 2.0 * s / vn2;
#pragma unroll
      for (int i = 0; i < 5; ++i) if (i >= k) b[i] -= s * A[3 * i + k];
    }
    A[3 * k + k] = alpha;
  }
  const double maxpiv = fmax(fmax(fabs(A[0]), fabs(A[4])), fabs(A[8]));
  const double thr = maxpiv * (3.0 * DBL_EPSILON);
  const int rank = (fabs(A[0]) > thr) + (fabs(A[4]) > thr) + (fabs(A[8]) > thr);
  double y[3] = {0, 0, 0};
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    if (k < rank) {
      double s = b[k];
#pragma unroll
      for (int j = 0; j < 3; ++j) if (j > k && j < rank) s -= A[3 * k + j] * y[j];
      y[k] = s / A[3 * k + k];
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) n[c] = perm[0] == c ? y[0] : (perm[1] == c ? y[1] : y[2]);   // n[perm[k]] = y[k]
}

}  // namespace

// K5: exact 5-NN of every stack point at pose7.  counts3 = {n_corner, n_surf, n_corner + n_surf} in device memory;
// query w < n_corner is corner point w, else surf point w - n_corner.  nbr[5 w + j] = j-th neighbour (x, y, z, index bits);
// nbr[5 w].w = -1 marks a query without an accepted neighbourhood (fewer than 5 points in reach, 5th farther than 1 m,
// or -- sharded -- a cell another rank owns).
__device__ __forceinline__ void map_knn5_body(const Pt4* __restrict__ corner_stack, const Pt4* __restrict__ surf_stack,
                                                  const int* __restrict__ counts3, MapCloud corner_map, MapCloud surf_map,
                                                  const double* __restrict__ pose7, float4* __restrict__ nbr, int shard_rank,
                                                  int shard_count) {
  pdl_launch_dependents();
  pdl_wait();   // pose7 is produced by the preceding LM solve of the stream
  const int n_corner = counts3[0], nq = counts3[2];
  const unsigned lane = lane_id();
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const unsigned mask_c = corner_map.grid.dyn->mask, mask_s = surf_map.grid.dyn->mask;
  double pose[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = pose7[k];
  for (int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; wid < nq; wid += warps) {
    const bool is_corner = wid < n_corner;
    const Pt4 ori = is_corner ? corner_stack[wid] : surf_stack[wid - n_corner];
    const GridTable& G = is_corner ? corner_map.grid : surf_map.grid;
    const Pt4 q = point_associate_to_map(ori, pose[0], pose[1], pose[2], pose[3], pose[4], pose[5], pose[6]);
    const float qx = q.x, qy = q.y, qz = q.z;
    bool reject = false;
    if (shard_count > 1 && owner_of(cell_of(qx, G.inv_cs), shard_count) != shard_rank) reject = true;
    float nd[5]; int ni[5], np[5];
    if (!reject) {
      TopK<5> t; t.init();
      visit_block27(G, is_corner ? mask_c : mask_s, qx, qy, qz,
                    [&](float x, float y, float z, int idx, int slot) { t.push(sqdist3(x, y, z, qx, qy, qz), idx, slot); });
      const int found = warp_merge_topk<5>(t, nd, ni, np);
      reject = !(found == 5 && (double)nd[4] < 1.0);   // pointSearchSqDis[4] < 1.0 (:584,652)
    }
    if (reject) {
      if (lane == 0) nbr[(size_t)wid * 5] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
    } else if (lane < 5) {
      int slot = np[0];
#pragma unroll
      for (int j = 1; j < 5; ++j) if ((int)lane == j) slot = np[j];
      nbr[(size_t)wid * 5 + lane] = __ldg(G.gpts + slot);
    }
  }
}
// grid (CTAs, 1, lanes)
__global__ void __launch_bounds__(256) k_map_knn5(const __grid_constant__ Batch<MapAssocArgs> B, int shard_rank, int shard_count) {
  const MapAssocArgs& a = B.a[blockIdx.z];
  map_knn5_body(a.corner_stack, a.surf_stack, a.counts3, a.corner_map, a.surf_map, a.pose7, a.nbr, shard_rank, shard_count);
}


// K5 against the prior map (localising lanes): k_map_knn5's search in the ONE grid over the whole frozen map, shared by all lanes.
// A candidate counts only if its cube lies in the lane's 5 x 5 x 3 window, and candidates are ordered by (distance, window offset
// of the cube + rank in the cube) -- the index the point would have had in the submap a mapping frame gathers from the same
// store.  So the five neighbours and their order are those of gather + K0 + k_map_knn5, and nbr (index bits included) is
// identical.  The window tables of the lane live in shared memory (600 B).
// grid (CTAs, 1, lanes)
__global__ void __launch_bounds__(256) k_map_knn5_prior(const __grid_constant__ Batch<MapPriorArgs> B, const __grid_constant__ PriorGrid P) {
  const MapPriorArgs& a = B.a[blockIdx.z];
  pdl_launch_dependents();
  pdl_wait();   // pose7 is produced by the preceding LM solve of the stream, the window by k_locate_begin
  __shared__ int s_win[2][ALOAM_WINDOW_CUBES];
  __shared__ int s_ctr[3];
  if (threadIdx.x < 2 * ALOAM_WINDOW_CUBES) s_win[threadIdx.x / ALOAM_WINDOW_CUBES][threadIdx.x % ALOAM_WINDOW_CUBES] = a.win[threadIdx.x / ALOAM_WINDOW_CUBES][threadIdx.x % ALOAM_WINDOW_CUBES];
  else if (threadIdx.x < 2 * ALOAM_WINDOW_CUBES + 3) s_ctr[threadIdx.x - 2 * ALOAM_WINDOW_CUBES] = a.ctr[threadIdx.x - 2 * ALOAM_WINDOW_CUBES];
  __syncthreads();
  const Pt4* __restrict__ corner_stack = a.corner_stack;
  const Pt4* __restrict__ surf_stack = a.surf_stack;
  float4* __restrict__ nbr = a.nbr;
  const int n_corner = a.counts3[0], nq = a.counts3[2];
  const unsigned lane = lane_id();
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const unsigned mask_c = P.corner.dyn->mask, mask_s = P.surf.dyn->mask;
  const int c0 = s_ctr[0] - 2, c1 = s_ctr[1] - 2, c2 = s_ctr[2] - 1;   // the window's low corner
  double pose[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = a.pose7[k];
  for (int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; wid < nq; wid += warps) {
    const bool is_corner = wid < n_corner;
    const Pt4 ori = is_corner ? corner_stack[wid] : surf_stack[wid - n_corner];
    const GridTable& G = is_corner ? P.corner : P.surf;
    const int* win = s_win[is_corner ? 0 : 1];
    const Pt4 q = point_associate_to_map(ori, pose[0], pose[1], pose[2], pose[3], pose[4], pose[5], pose[6]);
    const float qx = q.x, qy = q.y, qz = q.z;
    float nd[5]; int ni[5], np[5];
    TopK<5> t; t.init();
    visit_block27(G, is_corner ? mask_c : mask_s, qx, qy, qz, [&](float x, float y, float z, int tag, int slot) {
      const unsigned u = (unsigned)tag;   // i sets bit 31 from i = 16 on: decoded unsigned
      const int di = (int)(u >> 27) - c0, dj = (int)((u >> 22) & 31u) - c1, dk = (int)((u >> 18) & 15u) - c2;
      if ((unsigned)di < 5u && (unsigned)dj < 5u && (unsigned)dk < 3u)   // a cube of the window (one that holds points is inside the buffer)
        t.push(sqdist3(x, y, z, qx, qy, qz), win[(di * 5 + dj) * 3 + dk] + (int)(u & 0x3ffffu), slot);
    });
    const int found = warp_merge_topk<5>(t, nd, ni, np);
    if (!(found == 5 && (double)nd[4] < 1.0)) {   // pointSearchSqDis[4] < 1.0 (:584,652)
      if (lane == 0) nbr[(size_t)wid * 5] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
    } else if (lane < 5) {
      int slot = np[0], idx = ni[0];
#pragma unroll
      for (int j = 1; j < 5; ++j) if ((int)lane == j) { slot = np[j]; idx = ni[j]; }
      float4 p = __ldg(G.gpts + slot);
      p.w = __int_as_float(idx);
      nbr[(size_t)wid * 5 + lane] = p;
    }
  }
}


// K6: one thread per stack point: line fit (:586-621) or plane fit (:650-686) on its five neighbours, residual block out.
__device__ __forceinline__ void map_fit_body(const Pt4* __restrict__ corner_stack, const Pt4* __restrict__ surf_stack,
                                                 const int* __restrict__ counts3, const float4* __restrict__ nbr,
                                                 BlockRec* __restrict__ blocks, double* __restrict__ fits) {
  pdl_launch_dependents();
  pdl_wait();
  const int n_corner = counts3[0], nq = counts3[2];
  for (int wid = blockIdx.x * blockDim.x + threadIdx.x; wid < nq; wid += gridDim.x * blockDim.x) {
    const bool is_corner = wid < n_corner;
    BlockRec* out = blocks + wid;
    double* fo = fits ? fits + (size_t)wid * 14 : nullptr;
    const float4 n0 = nbr[(size_t)wid * 5];
    if (__float_as_int(n0.w) < 0) { out->type = -1; if (fo) fo[1] = -1.0; continue; }
    const Pt4 ori = is_corner ? corner_stack[wid] : surf_stack[wid - n_corner];
    double P[15];
    int ni[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float4 p = j == 0 ? n0 : nbr[(size_t)wid * 5 + j];
      P[3 * j] = p.x; P[3 * j + 1] = p.y; P[3 * j + 2] = p.z; ni[j] = __float_as_int(p.w);
    }
    out->cp[0] = ori.x; out->cp[1] = ori.y; out->cp[2] = ori.z;
    if (fo) { fo[0] = is_corner ? wid : wid - n_corner; for (int j = 0; j < 5; ++j) fo[9 + j] = ni[j]; }
    if (is_corner) {
      // :586-616  centre, scatter matrix, eigen-decomposition, line test
      double c[3] = {0, 0, 0};
#pragma unroll
      for (int j = 0; j < 5; ++j) { c[0] = c[0] + P[3 * j]; c[1] = c[1] + P[3 * j + 1]; c[2] = c[2] + P[3 * j + 2]; }
      c[0] = c[0] / 5.0; c[1] = c[1] / 5.0; c[2] = c[2] / 5.0;
      double cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const double d[3] = {P[3 * j] - c[0], P[3 * j + 1] - c[1], P[3 * j + 2] - c[2]};
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int b = 0; b < 3; ++b) cov[3 * a + b] += d[a] * d[b];
      }
      double ev[3], dir[3];
      eig3_sym(cov, ev, dir);
      if (!(ev[2] > 3 * ev[1])) { out->type = -1; if (fo) fo[1] = -1.0; continue; }
#pragma unroll
      for (int k = 0; k < 3; ++k) { out->a[k] = 0.1 * dir[k] + c[k]; out->b[k] = -0.1 * dir[k] + c[k]; }
      const double ex = out->a[0] - out->b[0], ey = out->a[1] - out->b[1], ez = out->a[2] - out->b[2];
      out->w = 1.0 / sqrt(ex * ex + ey * ey + ez * ez);
      out->s = 1.0;   // LidarEdgeFactor(curr_point, point_a, point_b, 1.0), laserMapping.cpp:618
      out->type = 0;
      if (fo) { fo[1] = 0.0; for (int k = 0; k < 3; ++k) { fo[2 + k] = out->a[k]; fo[5 + k] = out->b[k]; } fo[8] = 0.0; }
    } else {
      // :650-684  plane A n = -1, normalise, fit check, LidarPlaneNormFactor
      const double rhs[5] = {-1, -1, -1, -1, -1};
      double nv[3];
      lsq_5x3(P, rhs, nv);
      const double nn = sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
      const double neg_oa = 1 / nn;
      nv[0] /= nn; nv[1] /= nn; nv[2] /= nn;
      bool valid = true;
#pragma unroll
      for (int j = 0; j < 5; ++j)
        if (fabs(nv[0] * P[3 * j] + nv[1] * P[3 * j + 1] + nv[2] * P[3 * j + 2] + neg_oa) > 0.2) valid = false;
      if (!valid) { out->type = -1; if (fo) fo[1] = -1.0; continue; }
#pragma unroll
      for (int k = 0; k < 3; ++k) { out->a[k] = nv[k]; out->b[k] = 0.0; }
      out->s = neg_oa;
      out->w = 0.0;
      out->type = 2;
      if (fo) { fo[1] = 2.0; for (int k = 0; k < 3; ++k) { fo[2 + k] = nv[k]; fo[5 + k] = 0.0; } fo[8] = neg_oa; }
    }
  }
}
// grid (CTAs, 1, lanes)
__global__ void __launch_bounds__(128) k_map_fit(const __grid_constant__ Batch<MapAssocArgs> B) {
  const MapAssocArgs& a = B.a[blockIdx.z];
  map_fit_body(a.corner_stack, a.surf_stack, a.counts3, a.nbr, a.blocks, a.fits);
}


// exact k-NN (k <= 8) against a map cloud: 27-cell block first; if its k-th distance is not inside the guaranteed
// radius (one cell), a coalesced sweep over the whole (cell-sorted) cloud settles it
__global__ void __launch_bounds__(256) k_map_knn(MapCloud map, const Pt4* __restrict__ queries, int nq, int k,
                                                 int* __restrict__ idx, float* __restrict__ sqd) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wid >= nq) return;
  const Pt4 q = queries[wid];
  const int n = map.grid.dyn->n;
  TopK<8> t; t.init();
  visit_block27(map.grid, map.grid.dyn->mask, q.x, q.y, q.z,
                [&](float x, float y, float z, int i, int slot) { t.push(sqdist3(x, y, z, q.x, q.y, q.z), i, slot); });
  float od[8]; int oi[8], op[8];
  TopK<8> t2 = t;
  warp_merge_topk<8>(t2, od, oi, op);
  const float safe = map.grid.cs * map.grid.cs * 0.9999f;
  if (!(oi[k - 1] != INT_MAX && od[k - 1] < safe)) {
    t.init();
    for (int i = (int)lane_id(); i < n; i += 32) {
      const float4 p = map.grid.gpts[i];
      t.push(sqdist3(p.x, p.y, p.z, q.x, q.y, q.z), __float_as_int(p.w), i);
    }
    warp_merge_topk<8>(t, od, oi, op);
  }
  if (lane_id() == 0)
    for (int j = 0; j < k; ++j) {
      idx[(size_t)wid * k + j] = oi[j] == INT_MAX ? -1 : oi[j];
      sqd[(size_t)wid * k + j] = oi[j] == INT_MAX ? __int_as_float(0x7f800000) : od[j];
    }
}

}  // namespace aloam

// ---------------------------------------------------------------------------------------------------------------
// host side of the mapping entry points
using namespace aloam;

int comm_allreduce(aloam_ctx* c, const void* src, void* dst, size_t count, ncclDataType_t type);   // comm.cu

namespace {
inline int grid_ctas(const aloam_ctx* c) { return c->sms * 8; }   // grid-stride launches: 8 resident CTAs of 256 threads per SM

// device pointer with 16-byte points: the index can be built straight from the caller's memory (no staging copy)
bool is_device_ptr(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice;
}
}  // namespace

// the buffers of one registration set in g: the 5-NN records and residual blocks of `queries` points, the two stacks of
// queries / 2 points each and, with slots > 0, the two grid tables over submaps of up to `bound` points per type (`slots` slots
// each; a localising lane searches the prior map's and passes 0)
int map_reg_alloc(BufGroup& g, MapReg* r, size_t queries, size_t bound, unsigned slots) {
  for (int t = 0; t < 2 && slots > 0; ++t) {
    GridTable& gt = (t ? r->surf : r->corner).grid;
    if (!g.dev(&gt.slots, slots) || !g.dev(&gt.dyn, 1) || !g.dev(&gt.gpts, bound) || cudaMemset(gt.dyn, 0, sizeof(GridDyn)) != cudaSuccess)
      return ALOAM_ERR_CUDA;
    gt.cap_slots = slots;
    gt.cs = kMapCell;
    gt.inv_cs = 1.0f / gt.cs;
  }
  if (!g.dev(&r->nbr, queries * 5) || !g.dev(&r->blocks, queries) || !g.dev(&r->summary, 4) || !g.dev(&r->stack[0], queries / 2) ||
      !g.dev(&r->stack[1], queries / 2))
    return ALOAM_ERR_CUDA;
  return ALOAM_OK;
}

// the context's map buffers: the staging of uploaded maps, the registration set of the host API and mapper lane 0, and the
// host API's stack sizes, pose and fit records
int ensure_map_buffers(aloam_ctx* c) {
  if (c->map_ready) return ALOAM_OK;
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  c->max_map = c->cfg.max_map_points;
  unsigned slots = 1024;
  while (slots < (unsigned)c->max_map + ((unsigned)c->max_map >> 2)) slots <<= 1;   // ends: aloam_create bounds max_map_points by 2^30
  c->map_slots = (int)slots;
  const size_t mm = (size_t)c->max_map, mp = (size_t)c->max_points;
  BufGroup g;
  MapReg r = {};
  if (dalloc(c, &c->d_map_pts[0], mm) != cudaSuccess || dalloc(c, &c->d_map_pts[1], mm) != cudaSuccess || map_reg_alloc(g, &r, 2 * mp, mm, slots) != ALOAM_OK ||
      dalloc(c, &c->d_stack_counts, 4) != cudaSuccess || dalloc(c, &c->d_map_pose, 8) != cudaSuccess || dalloc(c, &c->d_fits, 2 * mp * 14) != cudaSuccess)
    return ALOAM_ERR_CUDA;
  own(c, std::move(g));
  c->map = r;
  c->map_ready = true;
  return ALOAM_OK;
}

// CTAs per lane of a grid-stride launch over nb lanes: one resident wave in all (8 CTAs of 256 threads per SM)
inline int lane_ctas(const aloam_ctx* c, int nb) { return std::max(1, grid_ctas(c) / nb); }

// K0 of nb lanes in one launch per phase: lane l indexes io[l].sub[0] / [1], already in device memory, into io[l].reg.  The
// clouds' sizes are in the GridDyn records (host upload: written by the caller; otherwise: k_grid_setup); n_upper bounds the
// larger cloud (grid sizing only).
void map_index_build(aloam_ctx* c, int nb, const MapLaneIO* io, int n_upper) {
  const int pb = std::max(1, std::min((std::max(n_upper, 1) + 255) / 256, lane_ctas(c, nb)));
  const unsigned slots_upper = grid_mask_for(std::max(n_upper, 1), (unsigned)c->map_slots) + 1;
  const int tb = std::max(1, std::min((int)((slots_upper + 255) / 256), lane_ctas(c, nb)));
  Batch<GridArgs> g = {};
  for (int l = 0; l < nb; ++l) g.a[l] = GridArgs{io[l].reg.corner.grid, io[l].sub[0], nullptr, io[l].reg.surf.grid, io[l].sub[1], nullptr};
  launch_ex(c, KID_MAP_GRID, k_grid_clear, dim3(tb, 1, nb), dim3(256), 0, 1, true, g);
  launch_ex(c, KID_MAP_GRID, k_grid_insert, dim3(pb, 2, nb), dim3(256), 0, 1, true, g, c->shard_rank, c->shard_count);
  launch_ex(c, KID_MAP_GRID, k_grid_alloc, dim3(tb, 1, nb), dim3(256), 0, 1, true, g);
  launch_ex(c, KID_MAP_GRID, k_grid_fill, dim3(pb, 2, nb), dim3(256), 0, 1, true, g);
}

namespace {
// 5-NN + fits of nb lanes, one launch each covering all of them: lane l associates io[l].reg.stack[0] / [1] (sizes io[l].counts3 =
// {n_corner, n_surf, total}) at pose io[l].pose with io[l].reg's submaps into its residual blocks, all in device memory.  fits:
// lane 0's debug records, or null.  pdl: the 5-NN may become resident under the previous kernel of the stream.
// prior: the lanes localise -- the 5-NN searches the prior map's grids through each lane's cube window instead of io[l].reg's.
void map_associate_device(aloam_ctx* c, int nb, const MapLaneIO* io, int nq_upper, bool pdl, double* fits, const PriorSearch* prior) {
  const int kb = std::max(1, std::min((nq_upper + 7) / 8, lane_ctas(c, nb)));
  const int fb = std::max(1, (nq_upper + 31) / 32);   // one warp per CTA: a few thousand serial double-precision fits spread over all SMs
  Batch<MapAssocArgs> a = {};
  for (int l = 0; l < nb; ++l)
    a.a[l] = MapAssocArgs{io[l].reg.stack[0], io[l].reg.stack[1], io[l].counts3, io[l].reg.corner, io[l].reg.surf, io[l].pose, io[l].reg.nbr,
                          io[l].reg.blocks, l == 0 ? fits : nullptr};
  if (prior) {
    Batch<MapPriorArgs> p = {};
    for (int l = 0; l < nb; ++l)
      p.a[l] = MapPriorArgs{io[l].reg.stack[0], io[l].reg.stack[1], io[l].counts3, io[l].pose, io[l].reg.nbr, {prior->win[l][0], prior->win[l][1]}, prior->ctr[l]};
    launch_ex(c, KID_MAP_KNN5_PRIOR, k_map_knn5_prior, dim3(kb, 1, nb), dim3(256), 0, 1, pdl, p, prior->grid);
  } else {
    launch_ex(c, KID_MAP_KNN5, k_map_knn5, dim3(kb, 1, nb), dim3(256), 0, 1, pdl, a, c->shard_rank, c->shard_count);
  }
  launch_ex(c, KID_MAP_FIT, k_map_fit, dim3(fb, 1, nb), dim3(32), 0, 1, true, a);
}
}  // namespace

// rounds x (5-NN + fits + LM) of nb lanes, each launch covering all of them: lane l registers its stacks against io[l].reg
// (see map_associate_device) and refines io[l].pose; round it leaves its summary in io[l].reg.summary[it & 3].  A sharded job's
// solves exchange their normal equations (one lane).
int map_register_device(aloam_ctx* c, int nb, const MapLaneIO* io, int nq_upper, int rounds, const PriorSearch* prior) {
  const LmParams lp = lm_params(c->cfg);
  for (int it = 0; it < rounds; ++it) {
    map_associate_device(c, nb, io, nq_upper, it > 0, nullptr, prior);
    Batch<LmArgs> lm = {};
    for (int l = 0; l < nb; ++l) lm.a[l] = LmArgs{io[l].reg.blocks, io[l].counts3 + 2, 0, io[l].pose, io[l].reg.summary + (it & 3), nullptr, nullptr};
    const int rc = launch_lm_batch(c, true, lm, nb, lp, 0, 0, false, sharded_lm(c));
    if (rc) return rc;
  }
  return ALOAM_OK;
}

namespace {
// One piece of cloud t of a sharded map cut into this rank's x-slabs + halo and appended to d_map_pts[t], behind the d_kept[t]
// points already there: the n points `stride` floats apart at pts, or only the first *n_dev of them when n_dev is set (a submap
// gathered on the device; n bounds it).  An overflow of max_map sets bit 0 of *err.
int shard_cut(aloam_ctx* c, int t, const float* pts, int stride, int n, const int* n_dev, int* d_kept, int* err) {
  int* d_blocks = reinterpret_cast<int*>(c->map.nbr);   // the per-block counts: scratch outside a registration
  const int nb = std::max(1, (n + 255) / 256);
  if ((size_t)nb * 4 > (size_t)2 * c->max_points * 5 * sizeof(float4)) return ALOAM_ERR_CAPACITY;
  const float inv_cs = c->map.corner.grid.inv_cs;
  LAUNCH(c, KID_MAP_GRID, k_shard_count, nb, 256, 0, pts, stride, n, n_dev, inv_cs, c->shard_rank, c->shard_count, d_blocks);
  LAUNCH(c, KID_MAP_GRID, k_shard_scan, 1, 1024, 0, d_blocks, nb, d_kept + t, c->max_map);
  LAUNCH(c, KID_MAP_GRID, k_shard_scatter, nb, 256, 0, pts, stride, n, n_dev, inv_cs, c->shard_rank, c->shard_count, (const int*)d_blocks,
         c->d_map_pts[t], c->max_map, err);
  return ALOAM_OK;
}

// K0 over the cut clouds d_map_pts[0] / [1] into the context's set; their sizes are d_kept[0] / [1] on the device
void shard_index(aloam_ctx* c, const int* d_kept) {
  const MapLaneIO io = {c->map, {c->d_map_pts[0], c->d_map_pts[1]}, nullptr, nullptr};
  Batch<GridArgs> g = {};
  g.a[0] = GridArgs{c->map.corner.grid, io.sub[0], d_kept, c->map.surf.grid, io.sub[1], d_kept + 1};
  LAUNCH(c, KID_MAP_GRID, k_grid_setup, 1, 32, 0, g);
  map_index_build(c, 1, &io, c->max_map);
}

// The end of both map uploads, once the index build is issued.  A rank of a sharded job sums the points in owned cells over the
// ranks: the thin-map test of laserMapping.cpp:554 is on the WHOLE submap, so every rank takes the same branch (a rank with a
// thin shard must still meet the others in the all-reduce).  Then the stream is synchronised and the map published.  kept,
// read after the synchronise: the points indexed on this rank (corner, surf) and the shard's overflow word.
int finish_map_upload(aloam_ctx* c, const int* kept) {
  if (c->shard_count > 1) {
    int* d_two = c->d_stack_counts;   // scratch: a sharded upload has copied its counts out of it before (stream order)
    CUDA_CHECK_RET(cudaMemcpyAsync(d_two, &c->map.corner.grid.dyn->owned, 4, cudaMemcpyDeviceToDevice, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(d_two + 1, &c->map.surf.grid.dyn->owned, 4, cudaMemcpyDeviceToDevice, c->stream));
    int rc = comm_allreduce(c, d_two, d_two, 2, ncclInt32); if (rc) return rc;
    CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->owned, d_two, 8, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  if (kept[2]) return ALOAM_ERR_CAPACITY;   // the shard does not fit cfg.max_map_points: the index holds a part of it, have_map stays false
  for (int t = 0; t < 2; ++t) { c->map_n[t] = kept[t]; c->map_global_n[t] = c->shard_count > 1 ? c->pin->owned[t] : kept[t]; }
  c->have_map = true;
  return ALOAM_OK;
}
}  // namespace

// The mapper of a rank of a sharded job (cubemap.cu): the gathered submap (whole, device-resident, sizes n_sub[0] / [1] on the
// device) is cut into this rank's x-slabs + halo and indexed, all in stream order -- nothing returns to the host.  An overflow
// of the shard buffer sets bit 0 of *err_word.
int map_shard_index_device(aloam_ctx* c, Pt4* const sub[2], const int* n_sub, int n_upper, int* err_word) {
  int* d_kept = c->d_stack_counts;    // [0], [1]: points kept per cloud (the mapper keeps its stack counts in its own state)
  CUDA_CHECK_RET(cudaMemsetAsync(d_kept, 0, 8, c->stream));
  for (int t = 0; t < 2; ++t) {
    const int rc = shard_cut(c, t, reinterpret_cast<const float*>(sub[t]), 4, n_upper, n_sub + t, d_kept, err_word);
    if (rc) return rc;
  }
  shard_index(c, d_kept);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

extern "C" {

int aloam_map_upload(aloam_ctx* c, aloam_cloud_view corner_map, aloam_cloud_view surf_map) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_map); if (rc) return rc;
  rc = check_view(surf_map); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  rc = ensure_map_buffers(c); if (rc) return rc;
  if (corner_map.n > c->max_map || surf_map.n > c->max_map) return ALOAM_ERR_CAPACITY;
  c->have_map = false;   // from here on the index is being rebuilt: published again by finish_map_upload
  // a 16-byte-stride cloud that already lives in device memory is indexed in place (the views are only borrowed for
  // the duration of this call: after the build nothing refers to the caller's memory, the cell-sorted copy is complete)
  const aloam_cloud_view views[2] = {corner_map, surf_map};
  const Pt4* src[2];
  for (int t = 0; t < 2; ++t) {
    if (views[t].n > 0 && views[t].stride_floats == 4 && is_device_ptr(views[t].data)) src[t] = reinterpret_cast<const Pt4*>(views[t].data);
    else { rc = upload_cloud(c, views[t], c->d_map_pts[t], c->max_map); if (rc) return rc; src[t] = c->d_map_pts[t]; }
  }
  GridDyn* hd = c->pin->grid;
  for (int t = 0; t < 2; ++t) { hd[t].n = views[t].n; hd[t].mask = grid_mask_for(views[t].n, (unsigned)c->map_slots); hd[t].cursor = 0; hd[t].owned = 0; }
  CUDA_CHECK_RET(cudaMemcpyAsync(c->map.corner.grid.dyn, &hd[0], sizeof(GridDyn), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->map.surf.grid.dyn, &hd[1], sizeof(GridDyn), cudaMemcpyHostToDevice, c->stream));
  const MapLaneIO io = {c->map, {src[0], src[1]}, nullptr, nullptr};
  map_index_build(c, 1, &io, std::max(corner_map.n, surf_map.n));
  const int kept[3] = {corner_map.n, surf_map.n, 0};
  return finish_map_upload(c, kept);
}

// aloam_map_upload for a rank of a sharded job that holds the WHOLE submap: the split into owned slabs + halo happens on the
// device (host views are streamed through in chunks), then the usual index build
int aloam_map_upload_sharded(aloam_ctx* c, aloam_cloud_view corner_map, aloam_cloud_view surf_map) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_map); if (rc) return rc;
  rc = check_view(surf_map); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  rc = ensure_map_buffers(c); if (rc) return rc;
  c->have_map = false;   // from here on the index is being rebuilt: published again by finish_map_upload
  const aloam_cloud_view views[2] = {corner_map, surf_map};
  int* d_kept = c->d_stack_counts;    // [0], [1]: points kept per cloud ; [2]: error word
  CUDA_CHECK_RET(cudaMemsetAsync(d_kept, 0, 16, c->stream));
  for (int t = 0; t < 2; ++t) {
    // a device view is cut in one piece, a host view goes through the corner stack buffer (max_points x 16 bytes) a chunk at a time
    const aloam_cloud_view v = views[t];
    const bool on_device = v.n > 0 && is_device_ptr(v.data);
    const int chunk = on_device ? v.n : std::max(1, c->max_points * 4 / std::max(v.stride_floats, 4));
    for (int off = 0; off < v.n; off += chunk) {
      const int m = std::min(chunk, v.n - off);
      const float* src = v.data;
      if (!on_device) {
        CUDA_CHECK_RET(cudaMemcpyAsync(c->map.stack[0], v.data + (size_t)off * v.stride_floats, (size_t)m * v.stride_floats * 4, cudaMemcpyHostToDevice, c->stream));
        src = reinterpret_cast<const float*>(c->map.stack[0]);
      }
      rc = shard_cut(c, t, src, v.stride_floats, m, nullptr, d_kept, d_kept + 2); if (rc) return rc;
    }
  }
  shard_index(c, d_kept);
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->shard, d_kept, 12, cudaMemcpyDeviceToHost, c->stream));
  return finish_map_upload(c, c->pin->shard);
}

int aloam_debug_map_sizes(aloam_ctx* c, int kept[2], int global[2]) {
  if (!c || !kept || !global) return ALOAM_ERR_INVALID_ARG;
  if (!c->have_map) return ALOAM_ERR_STATE;
  for (int t = 0; t < 2; ++t) { kept[t] = c->map_n[t]; global[t] = c->map_global_n[t]; }
  return ALOAM_OK;
}

static int upload_stacks(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack) {
  int rc = upload_cloud(c, corner_stack, c->map.stack[0], c->max_points); if (rc) return rc;
  rc = upload_cloud(c, surf_stack, c->map.stack[1], c->max_points); if (rc) return rc;
  int* sc = c->pin->stack_counts;
  sc[0] = corner_stack.n; sc[1] = surf_stack.n; sc[2] = corner_stack.n + surf_stack.n;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_stack_counts, sc, 12, cudaMemcpyHostToDevice, c->stream));
  return ALOAM_OK;
}

int aloam_mapping_register(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack, double x[7], aloam_stats* stats) {
  if (!c || !x) return ALOAM_ERR_INVALID_ARG;
  if (!c->have_map) return ALOAM_ERR_STATE;
  int rc = check_view(corner_stack); if (rc) return rc;
  rc = check_view(surf_stack); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (!(c->map_global_n[0] > 10 && c->map_global_n[1] > 50)) {   // laserMapping.cpp:554,730-733: pose unchanged
    if (stats) { std::memset(stats, 0, sizeof(*stats)); stats->flags = ALOAM_FLAG_MAP_TOO_THIN; }
    return ALOAM_OK;
  }
  CUDA_CHECK_RET(cudaEventRecord(c->ev0, c->stream));
  rc = upload_stacks(c, corner_stack, surf_stack); if (rc) return rc;
  for (int k = 0; k < 7; ++k) c->pin->pose_in[k] = x[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_map_pose, c->pin->pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  rc = peer_err_reset(c); if (rc) return rc;
  const MapLaneIO io = {c->map, {nullptr, nullptr}, c->d_stack_counts, c->d_map_pose};
  rc = map_register_device(c, 1, &io, corner_stack.n + surf_stack.n, c->cfg.outer_iters); if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->pose_out, c->d_map_pose, 56, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, c->map.summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, c->stream));
  rc = peer_err_fetch(c, &c->pin->peer_err); if (rc) return rc;
  CUDA_CHECK_RET(cudaEventRecord(c->ev1, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  for (int k = 0; k < 7; ++k) x[k] = c->pin->pose_out[k];
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  fill_stats(c, stats, c->cfg.outer_iters, 0, ms);
  return c->pin->peer_err ? ALOAM_ERR_COMM : ALOAM_OK;   // a peer did not answer: the pose rests on a partial sum
}

// association only (tests): the launches of one outer iteration of aloam_mapping_register through the context's registration
// set -- against its uploaded submaps, or with `prior` against the prior map through one lane's window.  fits = (n_corner +
// n_surf) x 14 doubles [query, type (-1 rejected), p0(3), p1(3), d, nn(5)].  The records start as NaN, so what a row leaves
// unwritten is NaN, the same on every call: a query without an accepted neighbourhood has only its type, one whose fit fails
// its type, query and nn.
static int associate_fits(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack, const double x[7], double* fits,
                          const PriorSearch* prior) {
  int rc = upload_stacks(c, corner_stack, surf_stack); if (rc) return rc;
  for (int k = 0; k < 7; ++k) c->pin->pose_in[k] = x[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_map_pose, c->pin->pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  const int nq = corner_stack.n + surf_stack.n;
  if (nq > 0) {
    CUDA_CHECK_RET(cudaMemsetAsync(c->d_fits, 0xff, (size_t)nq * 14 * 8, c->stream));
    const MapLaneIO io = {c->map, {nullptr, nullptr}, c->d_stack_counts, c->d_map_pose};
    map_associate_device(c, 1, &io, nq, false, c->d_fits, prior);
    CUDA_CHECK_RET(cudaMemcpyAsync(fits, c->d_fits, (size_t)nq * 14 * 8, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

int aloam_mapping_associate(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack, const double x[7], double* fits) {
  if (!c || !x || !fits) return ALOAM_ERR_INVALID_ARG;
  if (!c->have_map) return ALOAM_ERR_STATE;
  int rc = check_view(corner_stack); if (rc) return rc;
  rc = check_view(surf_stack); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  return associate_fits(c, corner_stack, surf_stack, x, fits, nullptr);
}

// aloam_mapping_associate against the prior map through the window of lane `lane`'s latest localising frame (tests)
int aloam_debug_prior_associate(aloam_ctx* c, int lane, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack, const double x[7],
                                double* fits) {
  if (!c || !x || !fits || lane < 0 || lane >= c->n_lanes) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_stack); if (rc) return rc;
  rc = check_view(surf_stack); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  PriorSearch ps;
  rc = locator_prior_search(c, lane, &ps); if (rc) return rc;
  rc = ensure_map_buffers(c); if (rc) return rc;   // the stacks, 5-NN records, residual blocks and fit records of the context's set
  return associate_fits(c, corner_stack, surf_stack, x, fits, &ps);
}

int aloam_map_knn_impl(aloam_ctx* c, int which, aloam_cloud_view queries, int k, int* idx, float* sqdist) {
  if (!c->have_map) return ALOAM_ERR_STATE;
  if (k < 1 || k > 8) return ALOAM_ERR_INVALID_ARG;
  int rc = upload_cloud(c, queries, c->d_query, c->max_points); if (rc) return rc;
  if (queries.n > 0) {
    if ((size_t)queries.n * k > (size_t)c->max_points) return ALOAM_ERR_CAPACITY;
    LAUNCH(c, KID_MAP_KNN, k_map_knn, (queries.n + 7) / 8, 256, 0, which == 2 ? c->map.corner : c->map.surf, c->d_query, queries.n, k,
           c->d_knn_idx, c->d_knn_d);
    CUDA_CHECK_RET(cudaMemcpyAsync(idx, c->d_knn_idx, (size_t)queries.n * k * 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(sqdist, c->d_knn_d, (size_t)queries.n * k * 4, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

}  // extern "C"
