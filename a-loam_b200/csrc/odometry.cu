// Scan-to-scan correspondence search on the GPU -- replaces laserOdometry.cpp:111-129 (TransformToStart),
// :299-483 (the two association loops) and :567-568 (the kd-tree builds).
//
// Index = a dense (azimuth bucket x ring) table per "last" cloud instead of a kd-tree (k_rab_* kernels): a counting
//   sort of the cloud into ALOAM_NB x W cells, bucket-major (W = the context's ring width, 64 or 128: every kernel here is a
//   template on it), so that "all rings of an azimuth bucket" and "rings rc-2..rc+2 of an azimuth bucket" are both contiguous
//   slices of one float4 array (x, y, z, index << log2 W | ring).
//   The order of points inside a cell depends on atomic timing, but every search below compares candidates on
//   (distance, original index / visiting rank), so results are a pure function of the input.
// Search = ONE WARP PER QUERY, exact.  The clouds live in the sensor frame of the last scan, so a point whose
//   azimuth differs from the query's by at least a has distance >= rho_q * sin(a) from it.  After buckets bq-k..bq+k
//   have been read a best distance below rho_q*sin(k*w) is final.  The kernel is bound by DEPENDENT L2 round trips
//   (cell table -> points -> decision), not by bytes, so the first sweep reads the whole interval bq-k0..bq+k0 at
//   once -- it is one contiguous slice of the bucket-major array: one round for its two delimiters, then 12 coalesced
//   float4 loads in flight per lane -- with k0 = 1 (3 for rho < 6.5 m, where a bucket is narrower than the point
//   spacing); 98 % of the queries end there.  The rest grow the interval bucket by bucket.  The sweep stops at the
//   latest when the bound exceeds the reference's own threshold (DISTANCE_SQ_THRESHOLD, 25 m^2 by default), beyond which
//   the reference discards the match anyway, or when the whole circle has been read.
// The 2nd / 3rd correspondence points of :312-361 / :402-455 use the same sweep restricted to the ring slice
// rc-dn..rc+up (rc-2..rc+2 at the default NEARBY_SCAN 2.5), with candidates ranked by the reference's visiting order
// (forward ascending first, then backward descending, strict '<'), so ties resolve exactly as the sequential loops do.
// "Ring" is int(intensity) = ring + 0.1 relTime truncated.  scanRegistration.cpp emits relTime in (-2, 6] (DESIGN.md
// section 3), so a cloud's int(intensity) is the physical ring or the one below and need not ascend: the invariant the search
// relies on is only  int_i >= max_{j<i} int_j - 1.  Under it (and NEARBY_SCAN >= 1) the loops' break indices do not depend on
// the closest point.  With up = the largest u with rc + u <= rc + NEARBY_SCAN and dn = the largest u with rc - u >=
// rc - NEARBY_SCAN (both in double, as the reference's int-vs-double tests; at most W) the forward break is the first index
// with int >= rc+up+1 and the backward break the last with int <= rc-dn-1, every candidate has int in rc-dn..rc+up, and the
// class and visiting rank of a candidate follow from (index vs closest, int vs rc) alone.
#include <climits>
#include <cfloat>
#include "common.cuh"
#include "kernels.h"

namespace aloam {

// validates a cloud handed in through the C ABI after its index is built: every int(intensity) is a legal ring and no
// earlier point has a ring two or more above (fwd_end[r + 2] is the first index with ring >= r + 2)
template <int W>
__global__ void k_ring_offsets(const Pt4* __restrict__ pts, int n, const int* __restrict__ fwd_end, int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = (int)pts[i].i;  // int(intensity) = scan line (laserOdometry.cpp:308,398)
  if (r < 0 || r > W - 1 || fwd_end[min(r + 2, W)] < i) atomicExch(err, 1);
}
template __global__ void k_ring_offsets<64>(const Pt4* __restrict__ pts, int n, const int* __restrict__ fwd_end, int* __restrict__ err);
template __global__ void k_ring_offsets<128>(const Pt4* __restrict__ pts, int n, const int* __restrict__ fwd_end, int* __restrict__ err);

// ---------------------------------------------------------------------------------------------------------------
// index build: counting sort of the cloud into (azimuth bucket, ring) cells, bucket-major
namespace {
constexpr float kPiF = 3.14159265358979f;
constexpr float kBucketW = 2.0f * kPiF / (float)ALOAM_NB;   // bucket width [rad]

__device__ __forceinline__ int bucket_of(float x, float y) {
  int b = (int)((atan2f(y, x) + kPiF) * ((float)ALOAM_NB / (2.0f * kPiF)));
  return min(max(b, 0), ALOAM_NB - 1);
}
}  // namespace

// log2 of the ring width: the ring bits of a packed word
template <int W> struct RingBits { static constexpr int value = W == 64 ? 6 : 7; static_assert(W == 64 || W == 128, "ring width"); };

// blockIdx.y selects the cloud (0 = a, 1 = b)
template <int W>
__global__ void k_rab_count(const __grid_constant__ Batch<RabArgs> B) {
  pdl_launch_dependents();   // the next kernel of the stream may become resident (it blocks in pdl_wait())
  const RabArgs& A = B.a[blockIdx.z];
  const RabIndex& g = blockIdx.y == 0 ? A.a : A.b;
  const Pt4* __restrict__ pts = blockIdx.y == 0 ? A.pa : A.pb;
  const int n = blockIdx.y == 0 ? *A.na : *A.nb;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Pt4 p = pts[i];
  const int ring = min(max((int)p.i, 0), W - 1);
  const int cell = bucket_of(p.x, p.y) * W + ring;
  g.cell_of[i] = cell;
  g.rank_of[i] = atomicAdd(&g.cnt[cell], 1);
  // first / last index of each ring: the lanes of a warp hold consecutive indices, so the lowest / highest lane of a ring's
  // group carries its smallest / largest index
  const unsigned grp = __match_any_sync(__activemask(), ring);
  const unsigned lane = lane_id();
  if (lane == (unsigned)(__ffs(grp) - 1)) atomicMin(&g.first_of[ring], i);
  if (lane == 31u - __clz(grp)) atomicMax(&g.last_of[ring], i);
}
template __global__ void k_rab_count<64>(const __grid_constant__ Batch<RabArgs> B);
template __global__ void k_rab_count<128>(const __grid_constant__ Batch<RabArgs> B);

// one CTA per cloud: exclusive scan of the ALOAM_NB*W cell counts -> start[], the break tables, and reset the scratch for
// the next build
template <int W>
__global__ void __launch_bounds__(1024) k_rab_scan(const __grid_constant__ Batch<RabArgs> B) {
  pdl_launch_dependents();
  pdl_wait();   // launched with a programmatic dependency on the previous kernel of the stream
  const RabIndex& g = blockIdx.x == 0 ? B.a[blockIdx.y].a : B.a[blockIdx.y].b;
  constexpr int NC = ALOAM_NB * W, PER = NC / 1024;
  __shared__ int s_w[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  // break tables, W / 32 ring entries per lane: warp 0 takes the suffix minima of first_of, warp 1 the prefix maxima of last_of
  if (W == 128) {   // four entries per lane, entry 32 k + lane in slot k; the carry runs across the slots
    if (w == 0) {
      const int n = blockIdx.x == 0 ? *B.a[blockIdx.y].na : *B.a[blockIdx.y].nb;
      int carry = n;   // min over the slots above, and n
#pragma unroll
      for (int k = W / 32 - 1; k >= 0; --k) {
        int v = g.first_of[32 * k + lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_down_sync(0xffffffffu, v, d); if (lane + d < 32) v = min(v, u); }
        g.fwd_end[32 * k + lane] = min(v, carry);
        carry = min(carry, __shfl_sync(0xffffffffu, v, 0));
      }
      if (lane == 0) g.fwd_end[W] = n;
    } else if (w == 1) {
      int carry = -1;   // max over the slots below
#pragma unroll
      for (int k = 0; k < W / 32; ++k) {
        int v = g.last_of[32 * k + lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v = max(v, u); }
        g.bwd_begin[1 + 32 * k + lane] = max(v, carry) + 1;
        carry = max(carry, __shfl_sync(0xffffffffu, v, 31));
      }
      if (lane == 0) g.bwd_begin[0] = 0;
    }
  } else if (w == 0) {   // W = 64: two entries per lane
    const int n = blockIdx.x == 0 ? *B.a[blockIdx.y].na : *B.a[blockIdx.y].nb;
    int lo = g.first_of[lane], hi = g.first_of[32 + lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_down_sync(0xffffffffu, hi, d); if (lane + d < 32) hi = min(hi, u); }
    const int hi_all = __shfl_sync(0xffffffffu, hi, 0);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_down_sync(0xffffffffu, lo, d); if (lane + d < 32) lo = min(lo, u); }
    g.fwd_end[lane] = min(min(lo, hi_all), n);
    g.fwd_end[32 + lane] = min(hi, n);
    if (lane == 0) g.fwd_end[64] = n;
  } else if (w == 1) {
    int lo = g.last_of[lane], hi = g.last_of[32 + lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, lo, d); if (lane >= d) lo = max(lo, u); }
    const int lo_all = __shfl_sync(0xffffffffu, lo, 31);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, hi, d); if (lane >= d) hi = max(hi, u); }
    // bwd_begin[r] = 1 + max(last_of[0 .. r-1]): the inclusive maxima shifted by one entry
    g.bwd_begin[1 + lane] = lo + 1;
    g.bwd_begin[33 + lane] = max(hi, lo_all) + 1;
    if (lane == 0) g.bwd_begin[0] = 0;
  }
  int v[PER], sum = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) { v[k] = g.cnt[t * PER + k]; g.cnt[t * PER + k] = 0; sum += v[k]; }
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
  }
  __syncthreads();
  if (t < W) { g.first_of[t] = INT_MAX; g.last_of[t] = -1; }   // every reader of the scratch is past the barriers above
  int run = s_w[w] + incl - sum;
#pragma unroll
  for (int k = 0; k < PER; ++k) { g.start[t * PER + k] = run; run += v[k]; }
  if (t == 1023) g.start[NC] = run;
}
template __global__ void k_rab_scan<64>(const __grid_constant__ Batch<RabArgs> B);
template __global__ void k_rab_scan<128>(const __grid_constant__ Batch<RabArgs> B);

template <int W>
__global__ void k_rab_fill(const __grid_constant__ Batch<RabArgs> B) {
  pdl_launch_dependents();
  pdl_wait();   // launched with a programmatic dependency on the previous kernel of the stream
  const RabArgs& A = B.a[blockIdx.z];
  const RabIndex& g = blockIdx.y == 0 ? A.a : A.b;
  const Pt4* __restrict__ pts = blockIdx.y == 0 ? A.pa : A.pb;
  const int n = blockIdx.y == 0 ? *A.na : *A.nb;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Pt4 p = pts[i];
  const int cell = g.cell_of[i];
  // index-major key: comparing keys compares indices, the reference's tie rule (the ring need not ascend with the index)
  // (i < 2^24 - 1 at W = 128, < 2^25 - 1 at W = 64: create_ctx bounds max_points, so the word stays below INT_MAX, the
  // search's "no candidate")
  g.gpts[g.start[cell] + g.rank_of[i]] = make_float4(p.x, p.y, p.z, __int_as_float((i << RingBits<W>::value) | (cell & (W - 1))));
}
template __global__ void k_rab_fill<64>(const __grid_constant__ Batch<RabArgs> B);
template __global__ void k_rab_fill<128>(const __grid_constant__ Batch<RabArgs> B);

// ---------------------------------------------------------------------------------------------------------------
// search
namespace {

// The visitors below are written for CODE SIZE as much as for loads in flight: every call site of the visitor lambda is
// inlined, the kernel is short enough to run on a cold instruction cache, and an earlier version with ~120 inlined copies
// of the lambda (13 k SASS instructions) spent more time fetching instructions than data.  Each helper has exactly one
// batch of B inlined copies inside a loop that is not unrolled.
//
// f(x, y, z, packed) over gpts[e0, e1) with B coalesced float4 loads in flight per lane.  Out-of-range slots are clamped
// to the last element, so a point may be visited more than once: every visitor in this file is idempotent (strict
// minimum on (d2, key)).
template <int B, typename F>
__device__ __forceinline__ void visit_span(const float4* __restrict__ gpts, int e0, int e1, F&& f) {
  if (e0 >= e1) return;
  const int lane = (int)lane_id(), last = e1 - 1;
#pragma unroll 1
  for (int base = e0; base < e1; base += 32 * B) {
    float4 p[B];
#pragma unroll
    for (int i = 0; i < B; ++i) p[i] = __ldg(gpts + min(base + lane + 32 * i, last));
#pragma unroll
    for (int i = 0; i < B; ++i) f(p[i].x, p[i].y, p[i].z, __float_as_int(p[i].w));
  }
}

// Ring slice [r_lo, r_hi] of azimuth buckets bq-k and bq+k (the two coincide when 2k == NB): the growth step of a sweep
// whose first interval was not enough (2 % of the queries).  (A variant that doubles the interval per step -- one
// delimiter round per step instead of two per bucket -- was tried: it shortens the rare far sweeps but its extra
// bookkeeping on the common path made the average launch slower; bucket-by-bucket growth stays.)
template <int W, typename F>
__device__ __forceinline__ void visit_ring_step(const RabIndex& g, int bq, int k, int r_lo, int r_hi, F&& f) {
  const int b0 = (bq - k + ALOAM_NB) % ALOAM_NB, b1 = (bq + k) % ALOAM_NB;
#pragma unroll 1
  for (int side = 0; side < 2; ++side) {
    if (side && b1 == b0) break;
    const int b = side ? b1 : b0;
    visit_span<4>(g.gpts, g.start[b * W + r_lo], g.start[b * W + r_hi + 1], f);
  }
}

// All rings of the azimuth buckets lo..hi (lo <= hi, indices may run past either end of the circle) are at most two
// contiguous slices of gpts: [a0, a1) and [b0, b1).  Their four delimiters are fetched in ONE round.
struct Spans2 { int a0, a1, b0, b1; };
template <int W>
__device__ __forceinline__ Spans2 bucket_interval(const RabIndex& g, int lo, int hi) {
  int c0, c1, c2 = 0, c3 = 0;
  if (hi - lo + 1 >= ALOAM_NB) { c0 = 0; c1 = ALOAM_NB * W; }
  else if (lo < 0) { c0 = (lo + ALOAM_NB) * W; c1 = ALOAM_NB * W; c3 = (hi + 1) * W; }
  else if (hi >= ALOAM_NB) { c0 = lo * W; c1 = ALOAM_NB * W; c3 = (hi - ALOAM_NB + 1) * W; }
  else { c0 = lo * W; c1 = (hi + 1) * W; }
  const int lane = (int)lane_id();
  const int v = g.start[lane == 0 ? c0 : lane == 1 ? c1 : lane == 2 ? c2 : c3];
  Spans2 s;
  s.a0 = __shfl_sync(0xffffffffu, v, 0); s.a1 = __shfl_sync(0xffffffffu, v, 1);
  s.b0 = __shfl_sync(0xffffffffu, v, 2); s.b1 = __shfl_sync(0xffffffffu, v, 3);
  return s;
}

// Ring slice [r_lo, r_hi] of each of the buckets bq-k..bq+k (k <= kMaxK0): 2k+1 short slices.  One round for all the
// delimiters, one round for the first 32 points of every slice, then whatever is left of slices longer than 32.
constexpr int kMaxK0 = 3;
template <int W, typename F>
__device__ __forceinline__ void visit_ring_slices(const RabIndex& g, int bq, int k, int r_lo, int r_hi, F&& f) {
  const int lane = (int)lane_id();
  const int nb = 2 * k + 1;
  int v = 0;
  if (lane < 2 * nb) {
    const int b = (bq - k + (lane >> 1) + ALOAM_NB) % ALOAM_NB;
    v = g.start[b * W + ((lane & 1) ? r_hi + 1 : r_lo)];
  }
  float4 p[2 * kMaxK0 + 1];
  unsigned valid = 0, longer = 0;
#pragma unroll
  for (int j = 0; j < 2 * kMaxK0 + 1; ++j) {
    const int e0 = __shfl_sync(0xffffffffu, v, 2 * j), e1 = __shfl_sync(0xffffffffu, v, 2 * j + 1);   // 0, 0 past nb
    if (e0 < e1) { p[j] = __ldg(g.gpts + min(e0 + lane, e1 - 1)); valid |= 1u << j; if (e1 - e0 > 32) longer |= 1u << j; }
  }
#pragma unroll
  for (int j = 0; j < 2 * kMaxK0 + 1; ++j)
    if (valid & (1u << j)) f(p[j].x, p[j].y, p[j].z, __float_as_int(p[j].w));
#pragma unroll 1
  while (longer) {
    const int j = __ffs(longer) - 1;
    longer &= longer - 1;
    visit_span<2>(g.gpts, __shfl_sync(0xffffffffu, v, 2 * j) + 32, __shfl_sync(0xffffffffu, v, 2 * j + 1), f);
  }
}

__device__ __forceinline__ int first_halfwidth(float rho) { return rho < 6.5f ? kMaxK0 : 1; }

// After buckets bq-k .. bq+k have been seen, every unseen point is at azimuth distance >= k*w from q, hence at
// distance >= rho_q * sin(k*w) (k*w < pi/2).  1e-4 rad absorbs atan2f / bucket rounding.  Returns the squared safe radius.
__device__ __forceinline__ float safe_radius_sq(float rho_q, int k) {
  // sin(a) >= a - a^3/6 for a >= 0: a LOWER bound is all the argument needs (and no libm call, whose large-argument slow
  // path costs a stack frame and ~1 k instructions of code); past 1.4 rad the polynomial's maximum 0.94 is used.
  const float a = fmaxf((float)k * kBucketW - 1e-4f, 0.f);
  const float s = a >= 1.4f ? 0.94f : a * (1.f - a * a * (1.f / 6.f));
  const float r = rho_q * s;
  return r * r * 0.9999f;
}

struct D3 { double x, y, z; };
__device__ __forceinline__ D3 cross3(const D3& a, const D3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

// laserOdometry.cpp:111-129.  s == 1 (DISTORTION 0): slerp(1, q) == q exactly; otherwise q_point_last = slerp(s, q) and
// t_point_last = s t.  Eigen q*v = v + w*uv + u x uv, uv = 2 u x v; double math, rounded to float on store (:125-127).
__device__ __forceinline__ void transform_to_start(const double* pose, double s, float px, float py, float pz, float& ox, float& oy, float& oz) {
  double qs[4] = {pose[0], pose[1], pose[2], pose[3]};
  double ts[3] = {pose[4], pose[5], pose[6]};
  if (s != 1.0) {
    slerp_identity(pose, s, qs);
    ts[0] = s * pose[4]; ts[1] = s * pose[5]; ts[2] = s * pose[6];
  }
  const D3 u{qs[0], qs[1], qs[2]};
  const double w = qs[3];
  const D3 v{(double)px, (double)py, (double)pz};
  D3 uv = cross3(u, v);
  uv.x = uv.x + uv.x; uv.y = uv.y + uv.y; uv.z = uv.z + uv.z;
  const D3 c2 = cross3(u, uv);
  ox = (float)(((v.x + w * uv.x) + c2.x) + ts[0]);
  oy = (float)(((v.y + w * uv.y) + c2.y) + ts[1]);
  oz = (float)(((v.z + w * uv.z) + c2.z) + ts[2]);
}
// interpolation ratio of a point of the current sweep (:113-118): float intensity minus its integer part, over SCAN_PERIOD
__device__ __forceinline__ double ratio_of(float intensity, int distortion) {
  return distortion ? (double)(intensity - (float)(int)intensity) / 0.1 : 1.0;
}

__device__ __forceinline__ void store_none(BlockRec* b, int* corr) {
  b->type = -1;
  if (corr) { corr[0] = -1; corr[1] = -1; corr[2] = -1; corr[3] = 0; }
}

constexpr int kBig = 1 << 25;       // separates forward ranks [0, 2^25 - 1) from backward ranks (create_ctx bounds max_points)

// exact nearest neighbour of q with d2 < limit (strict); returns its packed word (index << log2 W | ring) or -1, d2 in out_d,
// the half-width of the bucket interval it had to read in k_out.  Ties -> smaller index (packed order == index order).
template <int W>
__device__ __forceinline__ int rab_nearest(const RabIndex& g, float qx, float qy, float qz, float limit, float& out_d, int& k_out) {
  const int bq = bucket_of(qx, qy);
  const float rho = sqrtf(qx * qx + qy * qy);
  float best_d = limit; int best_i = INT_MAX;
  float wd = FLT_MAX; int wi = INT_MAX;
  auto f = [&](float x, float y, float z, int packed) {
    const float d2 = sqdist3(x, y, z, qx, qy, qz);
    if (d2 < best_d || (d2 == best_d && best_i != INT_MAX && packed < best_i)) { best_d = d2; best_i = packed; }
  };
  int k = first_halfwidth(rho);
  const Spans2 sp = bucket_interval<W>(g, bq - k, bq + k);
#pragma unroll 1
  for (int side = 0; side < 2; ++side) visit_span<12>(g.gpts, side ? sp.b0 : sp.a0, side ? sp.b1 : sp.a1, f);
#pragma unroll 1
  for (;;) {
    wd = best_i == INT_MAX ? FLT_MAX : best_d; wi = best_i;
    warp_argmin(wd, wi);
    const float safe2 = safe_radius_sq(rho, k);
    if ((wi != INT_MAX && wd < safe2) || safe2 >= limit || 2 * (k + 1) > ALOAM_NB) break;
    ++k;
    visit_ring_step<W>(g, bq, k, 0, W - 1, f);
  }
  k_out = k;
  out_d = wd;
  return (wi == INT_MAX || wd == FLT_MAX) ? -1 : wi;
}

}  // namespace

// W = 128 asks for one CTA per SM at least (minBlocks 1): without it ptxas keeps the 64-wide instance's 80 registers and spills
// 104 bytes; with it the instance takes 95 registers and no spill.  (minBlocks 0 leaves the 64-wide instance as it was.)
template <int W>
__global__ void __launch_bounds__(256, W == 128 ? 1 : 0) k_odom_assoc(const __grid_constant__ Batch<AssocArgs> B, OdomParams prm, int max_sharp) {
  constexpr int RB = RingBits<W>::value;
  pdl_launch_dependents();   // the LM solve that follows may become resident now; it blocks in its own pdl_wait()
  pdl_wait();                // the preceding LM solve (pose7 producer, blocks consumer) has completed
  const AssocArgs& A = B.a[blockIdx.y];   // blockIdx.y = trajectory of the batch
  const Pt4* __restrict__ sharp = A.sharp;
  const Pt4* __restrict__ flat = A.flat;
  const int* __restrict__ feat_counts = A.feat_counts;
  const LastCloud& corner = A.corner;
  const LastCloud& surf = A.surf;
  const double* __restrict__ pose7 = A.pose7;
  BlockRec* __restrict__ blocks = A.blocks;
  int* __restrict__ corr = A.corr;
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = lane_id();
  const bool is_corner = wid < max_sharp;
  const int qi = is_corner ? wid : wid - max_sharp;
  // one round for everything the setup needs: the query point is fetched before its slot is known to be in use (the
  // query buffers hold ALOAM_MAX_QUERIES points, every slot index is a valid address)
  const int nq = is_corner ? feat_counts[0] : feat_counts[2];
  const Pt4 cur = (is_corner ? sharp : flat)[min(qi, ALOAM_MAX_QUERIES - 1)];
  double pose[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = pose7[k];
  BlockRec* out = blocks + wid;
  int* co = corr ? corr + 4 * wid : nullptr;
  if (qi >= nq) { if (lane == 0) store_none(out, co); return; }
  const LastCloud& L = is_corner ? corner : surf;
  const RabIndex& g = L.index;
  float qx, qy, qz;
  const double s_ratio = ratio_of(cur.i, prm.distortion);
  transform_to_start(pose, s_ratio, cur.x, cur.y, cur.z, qx, qy, qz);
  // The reference compares a float distance with the DOUBLE threshold (:305,310,393,399).  thr is the smallest float whose
  // double value is >= it, so that d2 < thr holds for a float d2 exactly when (double)d2 < dist_sq_thresh: (float)25.3 rounds
  // below 25.3 and would reject a d2 of that float, which the reference accepts.  NaN stays NaN (no match), above FLT_MAX inf.
  float thr = (float)prm.dist_sq_thresh;
  if ((double)thr < prm.dist_sq_thresh) thr = nextafterf(thr, INFINITY);

  // nearest neighbour (kdtree*Last->nearestKSearch(pointSel, 1, ...), :302,390) then `< DISTANCE_SQ_THRESHOLD`
  float d1;
  int k_nn;
  const int packed1 = rab_nearest<W>(g, qx, qy, qz, thr, d1, k_nn);
  if (packed1 < 0 || !((double)d1 < prm.dist_sq_thresh)) { if (lane == 0) store_none(out, co); return; }
  const int closest = packed1 >> RB;
  const int rc = packed1 & (W - 1);   // closestPointScanID = int(intensity) of the closest point (k_rab_fill packs it)
  // rings rc-dn .. rc+up survive the break tests `int > rc + NEARBY_SCAN` / `int < rc - NEARBY_SCAN` (:319,345,405,433),
  // evaluated in double as the reference does.  The two sides are counted separately: rc + N and rc - N need not round
  // symmetrically (N = 3 - 2^-48 at rc = 32 keeps ring 35 but not ring 29).  W rings cover 0..W-1 from any rc, so the
  // bound makes a huge or infinite NEARBY_SCAN mean "never break", as in the reference.
  int up = 0; while (up < W && (double)(rc + up + 1) <= (double)rc + prm.nearby_scan) ++up;
  int dn = 0; while (dn < W && (double)(rc - dn - 1) >= (double)rc - prm.nearby_scan) ++dn;
  // the loops' ranges: forward (closest, fwd_end), backward [bwd_begin, closest).  Issued together with the closest point;
  // aloam_create guarantees NEARBY_SCAN >= 1, hence up, dn >= 1, which puts both break indices on the right side of `closest`.
  const int fwd_end = g.fwd_end[min(rc + up + 1, W)], bwd_begin = g.bwd_begin[max(rc - dn, 0)];
  const Pt4 pc = L.pts[closest];   // issued now, consumed after the second search

  // second search: class 2 / class 3 minima in the reference's visiting order (forward ascending, then backward descending).
  //   corner (:312-361): forward int > rc, backward int < rc; one class
  //   surf (:402-455):   class 2 = forward int <= rc, backward int >= rc; class 3 = the rest of the two ranges
  float b2 = thr, b3 = thr; int r2 = INT_MAX, r3 = INT_MAX;
  float w2 = FLT_MAX, w3 = FLT_MAX; int k2 = INT_MAX, k3 = INT_MAX;
  {
    const int bq = bucket_of(qx, qy);
    const float rho = sqrtf(qx * qx + qy * qy);
    const int r_lo = max(rc - dn, 0), r_hi = min(rc + up, W - 1);
    auto f = [&](float x, float y, float z, int packed) {
      const int idx = packed >> RB, ring = packed & (W - 1);
      if (idx == closest || idx >= fwd_end || idx < bwd_begin) return;
      const bool fwd = idx > closest;
      const bool same = fwd ? ring <= rc : ring >= rc;   // corner: skipped ; surf: class 2
      if (is_corner && same) return;
      const int rank = fwd ? (idx - closest) : (kBig + (closest - idx));
      const float d2 = sqdist3(x, y, z, qx, qy, qz);
      if (is_corner || same) { if (d2 < b2 || (d2 == b2 && r2 != INT_MAX && rank < r2)) { b2 = d2; r2 = rank; } }
      else { if (d2 < b3 || (d2 == b3 && r3 != INT_MAX && rank < r3)) { b3 = d2; r3 = rank; } }
    };
    int k = min(k_nn, kMaxK0);
    visit_ring_slices<W>(g, bq, k, r_lo, r_hi, f);
#pragma unroll 1
    for (;;) {
      w2 = r2 == INT_MAX ? FLT_MAX : b2; k2 = r2; warp_argmin(w2, k2);
      const float safe2 = safe_radius_sq(rho, k);
      bool done = k2 != INT_MAX && w2 < safe2;
      if (!is_corner) {
        w3 = r3 == INT_MAX ? FLT_MAX : b3; k3 = r3; warp_argmin(w3, k3);
        done = done && k3 != INT_MAX && w3 < safe2;
      }
      if (done || safe2 >= thr || 2 * (k + 1) > ALOAM_NB) break;
      ++k;
      visit_ring_step<W>(g, bq, k, r_lo, r_hi, f);
    }
  }
  // rank -> index
  int j2 = -1, j3 = -1;
  if (k2 != INT_MAX && w2 != FLT_MAX) j2 = k2 < kBig ? (closest + k2) : (closest - (k2 - kBig));
  if (!is_corner && k3 != INT_MAX && w3 != FLT_MAX) j3 = k3 < kBig ? (closest + k3) : (closest - (k3 - kBig));

  if (is_corner) {
    if (j2 < 0) { if (lane == 0) store_none(out, co); return; }
    if (lane == 0) {
      const Pt4 a = pc, b = L.pts[j2];
      out->cp[0] = cur.x; out->cp[1] = cur.y; out->cp[2] = cur.z;
      out->a[0] = a.x; out->a[1] = a.y; out->a[2] = a.z;
      out->b[0] = b.x; out->b[1] = b.y; out->b[2] = b.z;
      const double ex = (double)a.x - (double)b.x, ey = (double)a.y - (double)b.y, ez = (double)a.z - (double)b.z;
      out->w = 1.0 / sqrt(ex * ex + ey * ey + ez * ez);  // 1 / de.norm(), lidarFactor.hpp:36-40 (the LM kernel multiplies)
      out->s = s_ratio;
      out->type = 0;
      if (co) { co[0] = closest; co[1] = j2; co[2] = -1; co[3] = 1; }
    }
  } else {
    if (j2 < 0 || j3 < 0) { if (lane == 0) store_none(out, co); return; }
    if (lane == 0) {
      const Pt4 pj = pc, pl = L.pts[j2], pm = L.pts[j3];
      out->cp[0] = cur.x; out->cp[1] = cur.y; out->cp[2] = cur.z;
      out->a[0] = pj.x; out->a[1] = pj.y; out->a[2] = pj.z;
      // ljm_norm = (j - l) x (j - m), normalised (lidarFactor.hpp:64-65)
      const D3 jl{(double)pj.x - (double)pl.x, (double)pj.y - (double)pl.y, (double)pj.z - (double)pl.z};
      const D3 jm{(double)pj.x - (double)pm.x, (double)pj.y - (double)pm.y, (double)pj.z - (double)pm.z};
      D3 nrm = cross3(jl, jm);
      const double z = nrm.x * nrm.x + nrm.y * nrm.y + nrm.z * nrm.z;
      if (z > 0) { const double nn = sqrt(z); nrm.x /= nn; nrm.y /= nn; nrm.z /= nn; }
      out->b[0] = nrm.x; out->b[1] = nrm.y; out->b[2] = nrm.z;
      out->s = s_ratio;
      out->w = 0.0;
      out->type = 1;
      if (co) { co[0] = closest; co[1] = j2; co[2] = j3; co[3] = 1; }
    }
  }
}
template __global__ void k_odom_assoc<64>(const __grid_constant__ Batch<AssocArgs> B, OdomParams prm, int max_sharp);
template __global__ void k_odom_assoc<128>(const __grid_constant__ Batch<AssocArgs> B, OdomParams prm, int max_sharp);

// laserOdometry.cpp:133-148 TransformToEnd: undistort to the sweep start, then carry to the sweep end; the integer part of the
// intensity is kept (dead code in the reference -- its call sites are under `if (0)`, :533-552 -- offered through aloam_transform_to_end)
__global__ void k_transform_to_end(const Pt4* __restrict__ in, int n, const double* __restrict__ pose7, int distortion, Pt4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double pose[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = pose7[k];
  const Pt4 p = in[i];
  float ux, uy, uz;
  transform_to_start(pose, ratio_of(p.i, distortion), p.x, p.y, p.z, ux, uy, uz);
  // q_last_curr.inverse() = conjugate / squaredNorm (Eigen)
  const double n2 = pose[0] * pose[0] + pose[1] * pose[1] + pose[2] * pose[2] + pose[3] * pose[3];
  const D3 u{-pose[0] / n2, -pose[1] / n2, -pose[2] / n2};
  const double w = pose[3] / n2;
  const D3 v{(double)ux - pose[4], (double)uy - pose[5], (double)uz - pose[6]};
  D3 uv = cross3(u, v);
  uv.x = uv.x + uv.x; uv.y = uv.y + uv.y; uv.z = uv.z + uv.z;
  const D3 c2 = cross3(u, uv);
  Pt4 o;
  o.x = (float)((v.x + w * uv.x) + c2.x); o.y = (float)((v.y + w * uv.y) + c2.y); o.z = (float)((v.z + w * uv.z) + c2.z);
  o.i = (float)(int)p.i;
  out[i] = o;
}

// exact 1-NN of arbitrary queries against a "last" cloud (aloam_knn, which = 0/1): no distance limit
template <int W>
__global__ void __launch_bounds__(256) k_knn_last(LastCloud cloud, const Pt4* __restrict__ queries, int nq,
                                                  int* __restrict__ idx, float* __restrict__ sqd) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wid >= nq) return;
  const Pt4 q = queries[wid];
  float d;
  int k_used;
  const int packed = rab_nearest<W>(cloud.index, q.x, q.y, q.z, FLT_MAX, d, k_used);
  const int j = packed < 0 ? -1 : (packed >> RingBits<W>::value);
  if (lane_id() == 0) { idx[wid] = j; sqd[wid] = j < 0 ? __int_as_float(0x7f800000) : d; }
}
template __global__ void k_knn_last<64>(LastCloud cloud, const Pt4* __restrict__ queries, int nq, int* __restrict__ idx, float* __restrict__ sqd);
template __global__ void k_knn_last<128>(LastCloud cloud, const Pt4* __restrict__ queries, int nq, int* __restrict__ idx, float* __restrict__ sqd);

}  // namespace aloam
