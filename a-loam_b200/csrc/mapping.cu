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
#include "ctx.h"

namespace aloam {

namespace {
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kSlab = 8;  // cells per ownership slab (x direction)

__device__ __forceinline__ unsigned long long cell_key(int cx, int cy, int cz) {
  return ((unsigned long long)(unsigned)(cx + (1 << 20)) << 42) | ((unsigned long long)(unsigned)(cy + (1 << 20)) << 21) |
         (unsigned long long)(unsigned)(cz + (1 << 20));
}
__device__ __forceinline__ unsigned hash_key(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (unsigned)k;
}
__device__ __forceinline__ int cell_of(float v, float inv_cs) { return (int)floorf(v * inv_cs); }
__device__ __forceinline__ int owner_of(int cx, int count) {
  int slab = (cx + (1 << 20)) / kSlab;
  return slab % count;
}
__device__ __forceinline__ unsigned long long slot_key(const uint4& s) { return ((unsigned long long)s.y << 32) | s.x; }
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
__global__ void k_grid_setup(GridTable a, const int* __restrict__ na, GridTable b, const int* __restrict__ nb) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    a.dyn->n = *na; a.dyn->mask = min(table_mask_for(*na), a.cap_slots - 1); a.dyn->cursor = 0; a.dyn->owned = 0;
    b.dyn->n = *nb; b.dyn->mask = min(table_mask_for(*nb), b.cap_slots - 1); b.dyn->cursor = 0; b.dyn->owned = 0;
  }
}

__global__ void k_grid_clear(GridTable a, GridTable b) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gstride = gridDim.x * blockDim.x;
  const uint4 empty = make_uint4(~0u, ~0u, 0u, 0u);
  const int ma = (int)a.dyn->mask, mb = (int)b.dyn->mask;
  for (int i = gtid; i <= ma; i += gstride) a.slots[i] = empty;
  for (int i = gtid; i <= mb; i += gstride) b.slots[i] = empty;
}

// blockIdx.y selects the cloud (0 = a, 1 = b).  (Grouping the lanes of a cell with __match_any so that one lane claims the slot for
// the group was tried here and was slower -- the vote costs more than the atomics it saves; the fill below does profit from
// it.)
__global__ void k_grid_insert(GridTable a, const Pt4* __restrict__ pa, GridTable b, const Pt4* __restrict__ pb, int shard_rank,
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

// per-cell storage: block-wide exclusive scan of the counts, ONE atomicAdd per CTA and table on the cursor (a per-slot
// atomicAdd serialises ~500k updates of a single address for a 1M-point map).  Writes the cell's START
// into the `end` word; k_grid_fill advances it to the end.
__global__ void __launch_bounds__(256) k_grid_alloc(GridTable a, GridTable b) {
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

__global__ void k_grid_fill(GridTable a, const Pt4* __restrict__ pa, GridTable b, const Pt4* __restrict__ pb) {
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
__global__ void __launch_bounds__(1024) k_shard_scan(int* __restrict__ block_cnt, int nblocks, int* __restrict__ base_total) {
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
  if (t == 0) *base_total = s_carry;
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

__device__ __forceinline__ int warp_incl_scan(int v) {
  const unsigned lane = lane_id();
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= (unsigned)d) v += t;
  }
  return v;
}

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

// least squares A n = b (5x3) by Householder QR, fully unrolled (registers).  The oracle pivots columns (Eigen's
// colPivHouseholderQr); for a full-rank 5x3 system both give the least-squares solution to rounding (compared at 1e-10).
__device__ __forceinline__ void lsq_5x3(const double (&Ain)[15], const double (&bin)[5], double (&n)[3]) {
  double A[15], b[5];
#pragma unroll
  for (int i = 0; i < 15; ++i) A[i] = Ain[i];
#pragma unroll
  for (int i = 0; i < 5; ++i) b[i] = bin[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double norm2 = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) if (i >= k) norm2 += A[3 * i + k] * A[3 * i + k];
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
  n[2] = b[2] / A[8];
  n[1] = (b[1] - A[5] * n[2]) / A[4];
  n[0] = (b[0] - A[1] * n[1] - A[2] * n[2]) / A[0];
}

struct D3 { double x, y, z; };
__device__ __forceinline__ D3 cross3(const D3& a, const D3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

}  // namespace

// K5: exact 5-NN of every stack point at pose7.  counts3 = {n_corner, n_surf, n_corner + n_surf} in device memory;
// query w < n_corner is corner point w, else surf point w - n_corner.  nbr[5 w + j] = j-th neighbour (x, y, z, index bits);
// nbr[5 w].w = -1 marks a query without an accepted neighbourhood (fewer than 5 points in reach, 5th farther than 1 m,
// or -- sharded -- a cell another rank owns).
__global__ void __launch_bounds__(256) k_map_knn5(const Pt4* __restrict__ corner_stack, const Pt4* __restrict__ surf_stack,
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
    // pointAssociateToMap (:154-163): q * p + t in double, stored to float
    float qx, qy, qz;
    {
      const D3 u{pose[0], pose[1], pose[2]};
      const double w = pose[3];
      const D3 v{(double)ori.x, (double)ori.y, (double)ori.z};
      D3 uv = cross3(u, v);
      uv.x = uv.x + uv.x; uv.y = uv.y + uv.y; uv.z = uv.z + uv.z;
      const D3 c2 = cross3(u, uv);
      qx = (float)(((v.x + w * uv.x) + c2.x) + pose[4]);
      qy = (float)(((v.y + w * uv.y) + c2.y) + pose[5]);
      qz = (float)(((v.z + w * uv.z) + c2.z) + pose[6]);
    }
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

// K6: one thread per stack point: line fit (:586-621) or plane fit (:650-686) on its five neighbours, residual block out.
__global__ void __launch_bounds__(128) k_map_fit(const Pt4* __restrict__ corner_stack, const Pt4* __restrict__ surf_stack,
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

int comm_allreduce_int2(aloam_ctx* c, int* d_two);   // comm.cu

namespace {
inline int grid_ctas(const aloam_ctx* c) { return c->sms * 8; }   // grid-stride launches: 8 resident CTAs of 256 threads per SM

int ensure_map_buffers(aloam_ctx* c) {
  if (c->map_corner.grid.slots) return ALOAM_OK;
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  c->max_map = c->cfg.max_map_points;
  unsigned slots = 1024;
  while (slots < (unsigned)c->max_map + ((unsigned)c->max_map >> 2)) slots <<= 1;
  c->map_slots = (int)slots;
  const size_t mm = (size_t)c->max_map;
  for (int t = 0; t < 2; ++t) {
    MapCloud* m = t ? &c->map_surf : &c->map_corner;
    GridTable& g = m->grid;
    if (cudaMalloc((void**)&c->d_map_pts[t], mm * 16) != cudaSuccess || cudaMalloc((void**)&g.slots, (size_t)slots * 16) != cudaSuccess ||
        cudaMalloc((void**)&g.dyn, sizeof(GridDyn)) != cudaSuccess || cudaMalloc((void**)&g.gpts, mm * 16) != cudaSuccess)
      return ALOAM_ERR_CUDA;
    if (cudaMemset(g.dyn, 0, sizeof(GridDyn)) != cudaSuccess) return ALOAM_ERR_CUDA;
    g.cap_slots = slots;
    g.cs = 1.0f * (1.0f + 1e-5f);   // > 1 m so that an f32 d^2 < 1.0 neighbour can never sit outside the 27-cell block
    g.inv_cs = 1.0f / g.cs;
  }
  const size_t mp = (size_t)c->max_points;
  if (cudaMalloc((void**)&c->d_stack_corner, mp * 16) != cudaSuccess || cudaMalloc((void**)&c->d_stack_surf, mp * 16) != cudaSuccess ||
      cudaMalloc((void**)&c->d_fits, 2 * mp * 14 * 8) != cudaSuccess || cudaMalloc((void**)&c->d_map_blocks, 2 * mp * sizeof(BlockRec)) != cudaSuccess ||
      cudaMalloc((void**)&c->d_nbr, 2 * mp * 5 * sizeof(float4)) != cudaSuccess || cudaMalloc((void**)&c->d_stack_counts, 4 * sizeof(int)) != cudaSuccess ||
      cudaMalloc((void**)&c->d_map_pose, 8 * sizeof(double)) != cudaSuccess || cudaMalloc((void**)&c->d_map_summary, 4 * sizeof(LmSummary)) != cudaSuccess)
    return ALOAM_ERR_CUDA;
  return ALOAM_OK;
}

// device pointer with 16-byte points: the index can be built straight from the caller's memory (no staging copy)
bool is_device_ptr(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice;
}
}  // namespace

// K0 over two clouds already in device memory; their sizes are in the GridDyn records (host path: written by the caller;
// mapping loop: k_grid_setup).  n_upper bounds the larger cloud (grid sizing only).
void map_index_build(aloam_ctx* c, const Pt4* d_corner, const Pt4* d_surf, int n_upper) {
  const int pb = std::max(1, std::min((std::max(n_upper, 1) + 255) / 256, grid_ctas(c)));
  const unsigned slots_upper = grid_mask_for(std::max(n_upper, 1), (unsigned)c->map_slots) + 1;
  const int tb = std::max(1, std::min((int)((slots_upper + 255) / 256), grid_ctas(c)));
  launch_ex(c, KID_MAP_GRID, k_grid_clear, dim3(tb), dim3(256), 0, 1, true, c->map_corner.grid, c->map_surf.grid);
  launch_ex(c, KID_MAP_GRID, k_grid_insert, dim3(dim3(pb, 2)), dim3(256), 0, 1, true, c->map_corner.grid, d_corner, c->map_surf.grid, d_surf, c->shard_rank, c->shard_count);
  launch_ex(c, KID_MAP_GRID, k_grid_alloc, dim3(tb), dim3(256), 0, 1, true, c->map_corner.grid, c->map_surf.grid);
  launch_ex(c, KID_MAP_GRID, k_grid_fill, dim3(dim3(pb, 2)), dim3(256), 0, 1, true, c->map_corner.grid, d_corner, c->map_surf.grid, d_surf);
}

// outer_iters x (5-NN + fits + LM) with the stacks, their counts {n_corner, n_surf, total} and the pose all in device memory
void map_register_device(aloam_ctx* c, const Pt4* d_corner_stack, const Pt4* d_surf_stack, const int* d_counts3, int nq_upper,
                         double* d_pose, bool want_fits) {
  const LmParams lp = lm_params(c->cfg);
  const int kb = std::max(1, std::min((nq_upper + 7) / 8, grid_ctas(c)));
  const int fb = std::max(1, (nq_upper + 31) / 32);   // one warp per CTA: a few thousand serial double-precision fits spread over all SMs
  for (int it = 0; it < c->cfg.outer_iters; ++it) {
    launch_ex(c, KID_MAP_KNN5, k_map_knn5, dim3(kb), dim3(256), 0, 1, it > 0, d_corner_stack, d_surf_stack, d_counts3, c->map_corner, c->map_surf,
              (const double*)d_pose, c->d_nbr, c->shard_rank, c->shard_count);
    launch_ex(c, KID_MAP_FIT, k_map_fit, dim3(fb), dim3(32), 0, 1, true, d_corner_stack, d_surf_stack, d_counts3, (const float4*)c->d_nbr,
              c->d_map_blocks, want_fits ? c->d_fits : (double*)nullptr);
    if (c->shard_count <= 1)
      launch_lm(c, true, (const BlockRec*)c->d_map_blocks, d_counts3 + 2, 0, d_pose, lp, c->d_map_summary + (it & 3), 0, (double*)nullptr, (double*)nullptr, 0);
    else
      launch_lm_sharded(c, c->d_map_blocks, d_counts3 + 2, d_pose, lp, c->d_map_summary + (it & 3));
  }
}

// The mapper of a rank of a sharded job (cubemap.cu): the gathered submap (whole, device-resident, sizes on the device) is cut
// into this rank's x-slabs + halo and indexed, all in stream order -- nothing returns to the host.  An overflow of the shard
// buffer sets bit 0 of *err_word.
int map_shard_index_device(aloam_ctx* c, const Pt4* sub_corner, const int* n_corner, const Pt4* sub_surf, const int* n_surf, int n_upper, int* err_word) {
  const Pt4* subs[2] = {sub_corner, sub_surf};
  const int* ns[2] = {n_corner, n_surf};
  int* d_cnt = c->d_stack_counts;    // [0], [1]: points kept per cloud (the mapper keeps its stack counts in its own state)
  int* d_blocks = reinterpret_cast<int*>(c->d_nbr);
  const int nb = std::max(1, (n_upper + 255) / 256);
  if ((size_t)nb * 4 > (size_t)2 * c->max_points * 5 * sizeof(float4)) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaMemsetAsync(d_cnt, 0, 8, c->stream));
  const float inv_cs = c->map_corner.grid.inv_cs;
  for (int t = 0; t < 2; ++t) {
    LAUNCH(c, KID_MAP_GRID, k_shard_count, nb, 256, 0, reinterpret_cast<const float*>(subs[t]), 4, n_upper, ns[t], inv_cs, c->shard_rank, c->shard_count, d_blocks);
    LAUNCH(c, KID_MAP_GRID, k_shard_scan, 1, 1024, 0, d_blocks, nb, d_cnt + t);
    LAUNCH(c, KID_MAP_GRID, k_shard_scatter, nb, 256, 0, reinterpret_cast<const float*>(subs[t]), 4, n_upper, ns[t], inv_cs, c->shard_rank, c->shard_count, (const int*)d_blocks,
           c->d_map_pts[t], c->max_map, err_word);
  }
  LAUNCH(c, KID_MAP_GRID, k_grid_setup, 1, 32, 0, c->map_corner.grid, (const int*)d_cnt, c->map_surf.grid, (const int*)(d_cnt + 1));
  map_index_build(c, c->d_map_pts[0], c->d_map_pts[1], c->max_map);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

extern "C" {

void aloam_map_free_impl(aloam_ctx* c) {
  for (int t = 0; t < 2; ++t) {
    MapCloud* m = t ? &c->map_surf : &c->map_corner;
    void* ps[] = {c->d_map_pts[t], m->grid.slots, m->grid.dyn, m->grid.gpts};
    for (void* p : ps) if (p) cudaFree(p);
  }
  void* qs[] = {c->d_stack_corner, c->d_stack_surf, c->d_fits, c->d_map_blocks, c->d_nbr, c->d_stack_counts, c->d_map_pose, c->d_map_summary};
  for (void* p : qs) if (p) cudaFree(p);
}

int aloam_map_upload_impl(aloam_ctx* c, aloam_cloud_view corner_map, aloam_cloud_view surf_map) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_map); if (rc) return rc;
  rc = check_view(surf_map); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  rc = ensure_map_buffers(c); if (rc) return rc;
  if (corner_map.n > c->max_map || surf_map.n > c->max_map) return ALOAM_ERR_CAPACITY;
  // a 16-byte-stride cloud that already lives in device memory is indexed in place (the views are only borrowed for
  // the duration of this call: after the build nothing refers to the caller's memory, the cell-sorted copy is complete)
  const aloam_cloud_view views[2] = {corner_map, surf_map};
  const Pt4* src[2];
  for (int t = 0; t < 2; ++t) {
    if (views[t].n > 0 && views[t].stride_floats == 4 && is_device_ptr(views[t].data)) src[t] = reinterpret_cast<const Pt4*>(views[t].data);
    else { rc = upload_cloud(c, views[t], c->d_map_pts[t], c->max_map); if (rc) return rc; src[t] = c->d_map_pts[t]; }
  }
  GridDyn* hd = reinterpret_cast<GridDyn*>(c->h_ints + 64);
  for (int t = 0; t < 2; ++t) { hd[t].n = views[t].n; hd[t].mask = grid_mask_for(views[t].n, (unsigned)c->map_slots); hd[t].cursor = 0; hd[t].owned = 0; }
  CUDA_CHECK_RET(cudaMemcpyAsync(c->map_corner.grid.dyn, &hd[0], sizeof(GridDyn), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->map_surf.grid.dyn, &hd[1], sizeof(GridDyn), cudaMemcpyHostToDevice, c->stream));
  map_index_build(c, src[0], src[1], std::max(corner_map.n, surf_map.n));
  c->map_n[0] = corner_map.n; c->map_n[1] = surf_map.n;
  c->map_global_n[0] = corner_map.n; c->map_global_n[1] = surf_map.n;
  if (c->shard_count > 1) {
    // the thin-map test of laserMapping.cpp:554 is on the WHOLE submap: sum the points in owned cells over the ranks, so
    // that every rank takes the same branch (a rank with a thin shard must still meet the others in the all-reduce)
    int* d_two = c->d_stack_counts ? c->d_stack_counts : nullptr;
    CUDA_CHECK_RET(cudaMemcpyAsync(d_two, &c->map_corner.grid.dyn->owned, 4, cudaMemcpyDeviceToDevice, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(d_two + 1, &c->map_surf.grid.dyn->owned, 4, cudaMemcpyDeviceToDevice, c->stream));
    rc = comm_allreduce_int2(c, d_two); if (rc) return rc;
    CUDA_CHECK_RET(cudaMemcpyAsync(c->h_ints + 80, d_two, 8, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  if (c->shard_count > 1) { c->map_global_n[0] = c->h_ints[80]; c->map_global_n[1] = c->h_ints[81]; }
  prof_collect(c);
  c->have_map = true;
  return ALOAM_OK;
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
  const aloam_cloud_view views[2] = {corner_map, surf_map};
  // host views go through the stack staging buffer (max_points x 16 bytes), a chunk at a time
  const float inv_cs = c->map_corner.grid.inv_cs;
  int* d_cnt = c->d_stack_counts;    // [0], [1]: points kept per cloud ; [2]: error word
  CUDA_CHECK_RET(cudaMemsetAsync(d_cnt, 0, 16, c->stream));
  int* d_blocks = reinterpret_cast<int*>(c->d_nbr);   // scratch for the block counts (unused outside a registration)
  for (int t = 0; t < 2; ++t) {
    const aloam_cloud_view v = views[t];
    const bool on_device = v.n > 0 && is_device_ptr(v.data);
    const int chunk = std::max(1, c->max_points * 4 / std::max(v.stride_floats, 4));
    for (int off = 0; off < v.n; off += on_device ? v.n : chunk) {
      const int m = on_device ? v.n : std::min(chunk, v.n - off);
      const float* src;
      int stride = v.stride_floats;
      if (on_device) src = v.data;
      else {
        CUDA_CHECK_RET(cudaMemcpyAsync(c->d_stack_corner, v.data + (size_t)off * v.stride_floats, (size_t)m * v.stride_floats * 4, cudaMemcpyHostToDevice, c->stream));
        src = reinterpret_cast<const float*>(c->d_stack_corner);
      }
      const int nb = (m + 255) / 256;
      if ((size_t)nb * 4 > (size_t)2 * c->max_points * 5 * sizeof(float4)) return ALOAM_ERR_CAPACITY;
      LAUNCH(c, KID_MAP_GRID, k_shard_count, nb, 256, 0, src, stride, m, (const int*)nullptr, inv_cs, c->shard_rank, c->shard_count, d_blocks);
      LAUNCH(c, KID_MAP_GRID, k_shard_scan, 1, 1024, 0, d_blocks, nb, d_cnt + t);
      LAUNCH(c, KID_MAP_GRID, k_shard_scatter, nb, 256, 0, src, stride, m, (const int*)nullptr, inv_cs, c->shard_rank, c->shard_count, (const int*)d_blocks, c->d_map_pts[t], c->max_map, d_cnt + 2);
    }
  }
  LAUNCH(c, KID_MAP_GRID, k_grid_setup, 1, 32, 0, c->map_corner.grid, (const int*)d_cnt, c->map_surf.grid, (const int*)(d_cnt + 1));
  map_index_build(c, c->d_map_pts[0], c->d_map_pts[1], c->max_map);
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_ints + 84, d_cnt, 12, cudaMemcpyDeviceToHost, c->stream));
  if (c->shard_count > 1) {
    int* d_two = d_cnt + 2;   // reuse after the error word has been copied out (stream order)
    CUDA_CHECK_RET(cudaMemcpyAsync(d_two, &c->map_corner.grid.dyn->owned, 4, cudaMemcpyDeviceToDevice, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(d_two + 1, &c->map_surf.grid.dyn->owned, 4, cudaMemcpyDeviceToDevice, c->stream));
    rc = comm_allreduce_int2(c, d_two); if (rc) return rc;
    CUDA_CHECK_RET(cudaMemcpyAsync(c->h_ints + 80, d_two, 8, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  if (c->h_ints[86]) return ALOAM_ERR_CAPACITY;   // the shard does not fit cfg.max_map_points
  c->map_n[0] = c->h_ints[84]; c->map_n[1] = c->h_ints[85];
  c->map_global_n[0] = c->shard_count > 1 ? c->h_ints[80] : c->map_n[0];
  c->map_global_n[1] = c->shard_count > 1 ? c->h_ints[81] : c->map_n[1];
  c->have_map = true;
  return ALOAM_OK;
}

static int upload_stacks(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack) {
  int rc = upload_cloud(c, corner_stack, c->d_stack_corner, c->max_points); if (rc) return rc;
  rc = upload_cloud(c, surf_stack, c->d_stack_surf, c->max_points); if (rc) return rc;
  c->h_ints[96] = corner_stack.n; c->h_ints[97] = surf_stack.n; c->h_ints[98] = corner_stack.n + surf_stack.n;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_stack_counts, c->h_ints + 96, 12, cudaMemcpyHostToDevice, c->stream));
  return ALOAM_OK;
}

int aloam_mapping_register_impl(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack, double x[7], aloam_stats* stats) {
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
  for (int k = 0; k < 7; ++k) c->h_dbl[k] = x[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_map_pose, c->h_dbl, 56, cudaMemcpyHostToDevice, c->stream));
  map_register_device(c, c->d_stack_corner, c->d_stack_surf, c->d_stack_counts, corner_stack.n + surf_stack.n, c->d_map_pose, false);
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_dbl + 8, c->d_map_pose, 56, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, c->d_map_summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaEventRecord(c->ev1, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  for (int k = 0; k < 7; ++k) x[k] = c->h_dbl[8 + k];
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  fill_stats(c, stats, c->cfg.outer_iters, 0, ms);
  return ALOAM_OK;
}

// association only (tests): fits = (n_corner + n_surf) x 14 doubles [query, type (-1 rejected), p0(3), p1(3), d, nn(5)]
int aloam_mapping_associate(aloam_ctx* c, aloam_cloud_view corner_stack, aloam_cloud_view surf_stack, const double x[7], double* fits) {
  if (!c || !x || !fits) return ALOAM_ERR_INVALID_ARG;
  if (!c->have_map) return ALOAM_ERR_STATE;
  int rc = check_view(corner_stack); if (rc) return rc;
  rc = check_view(surf_stack); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  rc = upload_stacks(c, corner_stack, surf_stack); if (rc) return rc;
  for (int k = 0; k < 7; ++k) c->h_dbl[k] = x[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_map_pose, c->h_dbl, 56, cudaMemcpyHostToDevice, c->stream));
  const int nq = corner_stack.n + surf_stack.n;
  if (nq > 0) {
    LAUNCH(c, KID_MAP_KNN5, k_map_knn5, std::min((nq + 7) / 8, grid_ctas(c)), 256, 0, c->d_stack_corner, c->d_stack_surf, c->d_stack_counts, c->map_corner,
           c->map_surf, c->d_map_pose, c->d_nbr, c->shard_rank, c->shard_count);
    LAUNCH(c, KID_MAP_FIT, k_map_fit, (nq + 31) / 32, 32, 0, c->d_stack_corner, c->d_stack_surf, c->d_stack_counts, c->d_nbr, c->d_map_blocks, c->d_fits);
    CUDA_CHECK_RET(cudaMemcpyAsync(fits, c->d_fits, (size_t)nq * 14 * 8, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

int aloam_map_knn_impl(aloam_ctx* c, int which, aloam_cloud_view queries, int k, int* idx, float* sqdist) {
  if (!c->have_map) return ALOAM_ERR_STATE;
  if (k < 1 || k > 8) return ALOAM_ERR_INVALID_ARG;
  int rc = upload_cloud(c, queries, c->d_query, c->max_points); if (rc) return rc;
  if (queries.n > 0) {
    if ((size_t)queries.n * k > (size_t)c->max_points) return ALOAM_ERR_CAPACITY;
    LAUNCH(c, KID_MAP_KNN, k_map_knn, (queries.n + 7) / 8, 256, 0, which == 2 ? c->map_corner : c->map_surf, c->d_query, queries.n, k,
           c->d_knn_idx, c->d_knn_d);
    CUDA_CHECK_RET(cudaMemcpyAsync(idx, c->d_knn_idx, (size_t)queries.n * k * 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(sqdist, c->d_knn_d, (size_t)queries.n * k * 4, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

}  // extern "C"
