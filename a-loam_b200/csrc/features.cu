// Feature extraction on the GPU -- replaces scanRegistration.cpp:85-112,129-408.
//
//   k_classify   (thread / return)   NaN + minimum-range removal (:85-112,136-137), elevation -> ring id (:166-205),
//                                    sweep-start azimuth (:141), the return that flips `halfPassed` (:209-224, found
//                                    with a parallel min instead of the sequential state machine), per-block ring
//                                    histograms for the stable counting sort that replaces laserCloudScans[] (:240)
//   k_ring_scan  (one CTA)           histogram -> global offsets, scanStartInd/scanEndInd (:249-251), endOri (:142-153)
//   k_scatter    (thread / return)   relTime + intensity (:226-239), stable scatter into the ring-major cloud (:247-252)
//   k_ring_features (CTA / ring)     curvature (:256-266), per-sixth sort by (curvature, index) (:282-289), greedy
//                                    sharp / less-sharp / flat picks with neighbour suppression (:291-390), less-flat
//                                    gather (:392-398), pcl::VoxelGrid(0.2) (:401-407) -- all in shared memory
//   k_compact    (CTA / ring)        ring-ordered concatenation of the four feature clouds (:304-310,356,407)
//
// Everything here is float32 with the reference's evaluation order (compiled -fmad=false); ties in the two
// reference-internal unstable sorts are resolved by original index (SURVEY.md 8a note 4).
#include <climits>
#include <cfloat>
#include "common.cuh"
#include "kernels.h"

namespace aloam {

// debug time stamps (SM clock), taken only when a tool arms them with aloam_debug_feature_cycles(ctx, NULL): g_dbg_pick = ring 8:
// [0..3] one segment walk (entry, after the register loads, after the sharp walk, after the flat walk), [4..5] picks made,
// [6..7] after the speculative pass / after the re-run loop, [8..19] (start, end) of the six segment walks
__device__ long long g_dbg_pick[8 + 12];
__device__ int g_dbg_stamp = 0;

namespace {

constexpr int CT = 256;        // threads per CTA in classify / scatter
constexpr int CHUNK = 1024;    // returns per CTA (CT x 4)
constexpr int ITERS = CHUNK / CT;
constexpr double kPi = 3.14159265358979323846;  // M_PI

__device__ __forceinline__ bool point_ok(float x, float y, float z, float thres2) {
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;  // pcl::removeNaNFromPointCloud (:136)
  return !(x * x + y * y + z * z < thres2);                        // removeClosedPointCloud (:99)
}

// scanRegistration.cpp:166-205 ; returns -1 when the reference drops the return
__device__ __forceinline__ int ring_of(float x, float y, float z, int n_scans) {
  // :166 double atan / sqrt over float products, *180/M_PI in double, stored to float
  float angle = (float)(atan((double)z / sqrt((double)(x * x + y * y))) * 180.0 / kPi);
  int id;
  if (n_scans == 16) {
    id = (int)((double)((angle + 15.0f) / 2.0f) + 0.5);
    if (id > n_scans - 1 || id < 0) return -1;
  } else if (n_scans == 32) {
    id = (int)(((double)angle + 92.0 / 3.0) * 3.0 / 4.0);
    if (id > n_scans - 1 || id < 0) return -1;
  } else {
    if ((double)angle >= -8.83) id = (int)((double)(2.0f - angle) * 3.0 + 0.5);
    else id = n_scans / 2 + (int)((-8.83 - (double)angle) * 2.0 + 0.5);
    if (angle > 2.0f || (double)angle < -24.33 || id > 50 || id < 0) return -1;
  }
  return id;
}

__device__ __forceinline__ void load_xyz(const float* __restrict__ raw, int i, int stride, float& x, float& y, float& z) {
  if (stride == 4) {
    float4 v = __ldg(reinterpret_cast<const float4*>(raw) + i);
    x = v.x; y = v.y; z = v.z;
  } else {
    const float* p = raw + (size_t)i * stride;
    x = __ldg(p); y = __ldg(p + 1); z = __ldg(p + 2);
  }
}

// azimuth of a return before the halfPassed flip (:208-218)
__device__ __forceinline__ float ori_first_half(float x, float y, float start_ori) {
  float ori = -atan2f(y, x);
  if ((double)ori < (double)start_ori - kPi / 2) ori = (float)((double)ori + 2 * kPi);
  else if ((double)ori > (double)start_ori + kPi * 3 / 2) ori = (float)((double)ori - 2 * kPi);
  return ori;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CT) k_classify(const __grid_constant__ Batch<ClassifyArgs> B, int n_scans, float thres2) {
  pdl_launch_dependents();   // the next kernel of the stream may become resident (it blocks in pdl_wait())
  // blockIdx.y = trajectory (lane) of the batch; a lane with fewer returns than the largest one has idle trailing CTAs
  const ClassifyArgs& A = B.a[blockIdx.y];
  const float* __restrict__ raw = A.raw;
  const int n = A.n, stride = A.stride;
  int8_t* __restrict__ ring_out = A.ring_out;
  int* __restrict__ hist = A.hist;
  ScanScalars* __restrict__ sc = A.sc;
  if (blockIdx.x * CHUNK >= n && blockIdx.x > 0) return;
  __shared__ int s_hist[64];
  __shared__ int s_first, s_last, s_half;
  const int tid = threadIdx.x;
  if (tid < 64) s_hist[tid] = 0;
  if (tid == 0) { s_first = INT_MAX; s_last = -1; s_half = INT_MAX; }
  __syncthreads();
  // every CTA finds the first surviving return itself (normally raw[0]) so start_ori needs no grid-wide step
  for (int base = 0; base < n; base += CT) {
    int i = base + tid;
    if (i < n) {
      float x, y, z; load_xyz(raw, i, stride, x, y, z);
      if (point_ok(x, y, z, thres2)) atomicMin(&s_first, i);
    }
    __syncthreads();
    int f = s_first;
    __syncthreads();
    if (f != INT_MAX) break;
  }
  const int first = s_first;
  float start_ori = 0.f;
  if (first != INT_MAX) {
    float x, y, z; load_xyz(raw, first, stride, x, y, z);
    start_ori = -atan2f(y, x);  // :141
  }
  int my_last = -1, my_half = INT_MAX;
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    int i = blockIdx.x * CHUNK + it * CT + tid;
    if (i >= n) continue;
    float x, y, z; load_xyz(raw, i, stride, x, y, z);
    int ring = -2;
    if (point_ok(x, y, z, thres2)) {
      my_last = max(my_last, i);
      ring = ring_of(x, y, z, n_scans);
      if (ring >= 0) {
        atomicAdd(&s_hist[ring], 1);
        float ori = ori_first_half(x, y, start_ori);
        if ((double)(ori - start_ori) > kPi) my_half = min(my_half, i);  // :220
      }
    }
    ring_out[i] = (int8_t)ring;
  }
  if (my_last >= 0) atomicMax(&s_last, my_last);
  if (my_half != INT_MAX) atomicMin(&s_half, my_half);
  __syncthreads();
  if (tid < 64) hist[blockIdx.x * 64 + tid] = s_hist[tid];
  if (tid == 0) {
    if (s_last >= 0) atomicMax(&sc->last_valid, s_last);
    if (s_half != INT_MAX) atomicMin(&sc->half_idx, s_half);
    if (blockIdx.x == 0) { sc->first_valid = first; sc->start_ori = start_ori; }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// one CTA of 1024 threads: thread (r = t>>4, s = t&15) owns slice s of ring r's per-block histogram column
__global__ void __launch_bounds__(1024) k_ring_scan(const __grid_constant__ Batch<RingScanArgs> B, int n_scans) {
  pdl_launch_dependents();
  pdl_wait();   // launched with a programmatic dependency on the previous kernel of the stream
  const RingScanArgs& A = B.a[blockIdx.x];   // one CTA per trajectory of the batch
  const float* __restrict__ raw = A.raw;
  const int stride = A.stride, nblocks = A.nblocks;
  const int* __restrict__ hist = A.hist;
  int* __restrict__ offsets = A.offsets;
  int* __restrict__ ring_start = A.ring_start;
  int* __restrict__ scan_start = A.scan_start;
  int* __restrict__ scan_end = A.scan_end;
  ScanScalars* __restrict__ sc = A.sc;
  ScanScalars* __restrict__ sc_next = A.sc_next;
  __shared__ int s_tot[64];
  __shared__ int s_start[65];
  const int t = threadIdx.x, r = t >> 4, s = t & 15;
  const int bps = (nblocks + 15) / 16;
  const int b0 = min(nblocks, s * bps), b1 = min(nblocks, b0 + bps);
  int local = 0;
  for (int b = b0; b < b1; ++b) local += hist[b * 64 + r];
  // inclusive scan across the 16 slices (half-warp)
  int incl = local;
#pragma unroll
  for (int d = 1; d < 16; d <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, d, 16);
    if (s >= d) incl += v;
  }
  if (s == 15) s_tot[r] = incl;
  __syncthreads();
  if (t < 32) {  // exclusive scan of 64 ring totals, two per lane
    int a = s_tot[2 * t], b = s_tot[2 * t + 1];
    int pair = a + b, inc = pair;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, inc, d);
      if (t >= d) inc += v;
    }
    int ex = inc - pair;
    s_start[2 * t] = ex;
    s_start[2 * t + 1] = ex + a;
    if (t == 31) s_start[64] = inc;
  }
  __syncthreads();
  int running = s_start[r] + (incl - local);
  for (int b = b0; b < b1; ++b) {
    offsets[b * 64 + r] = running;
    running += hist[b * 64 + r];
  }
  if (t <= 64) ring_start[t] = s_start[t];
  if (t < 64) {  // :249-251
    scan_start[t] = s_start[t] + 5;
    scan_end[t] = s_start[t + 1] - 6;
  }
  if (t == 0) {
    sc->n_full = s_start[64];
    float end_ori = 0.f;
    if (sc->last_valid >= 0) {
      float x, y, z; load_xyz(raw, sc->last_valid, stride, x, y, z);
      const float start_ori = sc->start_ori;
      end_ori = (float)((double)(-atan2f(y, x)) + 2 * kPi);  // :142-144
      if ((double)(end_ori - start_ori) > 3 * kPi) end_ori = (float)((double)end_ori - 2 * kPi);
      else if ((double)(end_ori - start_ori) < kPi) end_ori = (float)((double)end_ori + 2 * kPi);
    }
    sc->end_ori = end_ori;
    if (A.n_full_out) *A.n_full_out = s_start[64];   // per-scan record of a stream call (0 = nothing survived the filters)
    // arm the other parity slot for the next scan
    sc_next->first_valid = INT_MAX; sc_next->last_valid = -1; sc_next->half_idx = INT_MAX; sc_next->n_full = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CT) k_scatter(const __grid_constant__ Batch<ScatterArgs> B) {
  pdl_launch_dependents();
  pdl_wait();   // launched with a programmatic dependency on the previous kernel of the stream
  const ScatterArgs& A = B.a[blockIdx.y];
  const float* __restrict__ raw = A.raw;
  const int n = A.n, stride = A.stride;
  const int8_t* __restrict__ ring_in = A.ring_in;
  const int* __restrict__ offsets = A.offsets;
  const ScanScalars* __restrict__ sc = A.sc;
  Pt4* __restrict__ full = A.full;
  if (blockIdx.x * CHUNK >= n) return;
  __shared__ int s_cnt[ITERS * (CT / 32)][64];  // [slot = it*8 + warp][ring], then exclusive prefix over slots
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  for (int k = tid; k < ITERS * (CT / 32) * 64; k += CT) (&s_cnt[0][0])[k] = 0;
  __syncthreads();
  int ring[ITERS], rank[ITERS];
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    int i = blockIdx.x * CHUNK + it * CT + tid;
    int r = (i < n) ? (int)ring_in[i] : -2;
    ring[it] = r;
    unsigned grp = __match_any_sync(0xffffffffu, r);
    rank[it] = __popc(grp & ((1u << lane) - 1u));
    if (r >= 0 && rank[it] == 0) s_cnt[it * (CT / 32) + w][r] = __popc(grp);
  }
  __syncthreads();
  if (tid < 64) {
    int run = offsets[blockIdx.x * 64 + tid];
#pragma unroll
    for (int k = 0; k < ITERS * (CT / 32); ++k) { int c = s_cnt[k][tid]; s_cnt[k][tid] = run; run += c; }
  }
  __syncthreads();
  const float start_ori = sc->start_ori, end_ori = sc->end_ori;
  const int half_idx = sc->half_idx;
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    const int r = ring[it];
    if (r < 0) continue;
    int i = blockIdx.x * CHUNK + it * CT + tid;
    float x, y, z; load_xyz(raw, i, stride, x, y, z);
    float ori;
    if (i <= half_idx) {           // the flipping return itself still takes the first branch (:209-224)
      ori = ori_first_half(x, y, start_ori);
    } else {                       // :226-236
      ori = (float)((double)(-atan2f(y, x)) + 2 * kPi);
      if ((double)ori < (double)end_ori - kPi * 3 / 2) ori = (float)((double)ori + 2 * kPi);
      else if ((double)ori > (double)end_ori + kPi / 2) ori = (float)((double)ori - 2 * kPi);
    }
    float rel = (ori - start_ori) / (end_ori - start_ori);  // :238
    Pt4 p; p.x = x; p.y = y; p.z = z;
    p.i = (float)((double)r + 0.1 * (double)rel);           // :239 scanID + scanPeriod * relTime
    full[s_cnt[it * (CT / 32) + w][r] + rank[it]] = p;
  }
}

// ---------------------------------------------------------------------------------------------------------------
namespace {

// Bitonic sort of NT*E 64-bit keys held E per thread (element index i = t*E + s).  Compare-exchange partners at
// distance j live in the same thread (j < E: registers), in another lane of the warp (E <= j < 32E: shuffles) or in
// another warp (j >= 32E: one shared-memory exchange, conflict-free [slot][thread] layout).  For 2048 keys on 256
// threads that is 30 register + 30 shuffle + 6 shared-memory passes instead of 66 shared-memory passes.
template <int E, int NT>
__device__ __forceinline__ void hybrid_bitonic(unsigned long long (&v)[E], unsigned long long* buf) {
  const int t = (NT == 32) ? (int)(threadIdx.x & 31) : (int)threadIdx.x;
  constexpr int P = E * NT;
#pragma unroll 1
  for (int k = 2; k <= P; k <<= 1) {
#pragma unroll 1
    for (int j = k >> 1; j >= E; j >>= 1) {
      const int tx = j / E;  // partner thread = t ^ tx, same slot
      if (NT > 32 && tx >= 32) {
#pragma unroll
        for (int s2 = 0; s2 < E; ++s2) buf[s2 * NT + t] = v[s2];
        __syncthreads();
#pragma unroll
        for (int s2 = 0; s2 < E; ++s2) {
          const unsigned long long o = buf[s2 * NT + (t ^ tx)];
          const int i = t * E + s2;
          const bool keep_min = ((i & j) == 0) == ((i & k) == 0);
          v[s2] = keep_min ? (v[s2] < o ? v[s2] : o) : (v[s2] > o ? v[s2] : o);
        }
        __syncthreads();
      } else {
#pragma unroll
        for (int s2 = 0; s2 < E; ++s2) {
          const unsigned long long o = __shfl_xor_sync(0xffffffffu, v[s2], tx);
          const int i = t * E + s2;
          const bool keep_min = ((i & j) == 0) == ((i & k) == 0);
          v[s2] = keep_min ? (v[s2] < o ? v[s2] : o) : (v[s2] > o ? v[s2] : o);
        }
      }
    }
#pragma unroll
    for (int jj = E / 2; jj >= 1; jj >>= 1) {
      if (jj < k) {
#pragma unroll
        for (int s2 = 0; s2 < E; ++s2) {
          if ((s2 & jj) == 0) {
            const int i = t * E + s2;
            const bool up = (i & k) == 0;
            const unsigned long long x = v[s2], y = v[s2 | jj];
            if ((x > y) == up) { v[s2] = y; v[s2 | jj] = x; }
          }
        }
      }
    }
  }
}

// one warp sorts the curvature keys of one sixth of a ring (scanRegistration.cpp:288) and leaves them in out[0..len)
template <int E>
__device__ __forceinline__ void warp_sort_segment(const float* curv, int sp, int len, unsigned long long* out) {
  const int lane = threadIdx.x & 31;
  unsigned long long v[E];
#pragma unroll
  for (int s2 = 0; s2 < E; ++s2) {
    const int m = lane * E + s2;
    v[s2] = m < len ? (((unsigned long long)__float_as_uint(curv[sp + m]) << 12) | (unsigned)(sp + m)) : ~0ull;
  }
  hybrid_bitonic<E, 32>(v, nullptr);
#pragma unroll
  for (int s2 = 0; s2 < E; ++s2) {
    const int m = lane * E + s2;
    if (m < len) out[m] = v[s2];
  }
}

// the whole CTA (NT threads) sorts P = NT*E voxel keys ; key_of(i) supplies the key of slot i ; result in keys[0..P)
template <int E, int NT, typename KeyOf>
__device__ __forceinline__ void cta_sort_keys(unsigned long long* keys, KeyOf&& key_of) {
  const int t = threadIdx.x;
  unsigned long long v[E];
#pragma unroll
  for (int s2 = 0; s2 < E; ++s2) v[s2] = key_of(t * E + s2);
  hybrid_bitonic<E, NT>(v, keys);
#pragma unroll
  for (int s2 = 0; s2 < E; ++s2) keys[t * E + s2] = v[s2];
  __syncthreads();
}

// Merge sort of P = NT*E 64-bit keys by the whole CTA: every warp sorts its 32*E keys in registers / shuffles (the bitonic network
// above on one warp), then log2(NT/32) merge levels over two shared-memory buffers: every thread owns E consecutive outputs of a
// merged pair, finds where they start in the two runs with a merge-path binary search and merges E keys sequentially.
// 2048 keys on 512 threads: 28 warp-local stages + 4 levels of (11-step search + 4 picks), against 66 CTA-wide bitonic stages of
// which 10 go through shared memory with two barriers each.  Returns the buffer that holds the sorted keys.
template <int E, int NT, typename KeyOf>
__device__ __forceinline__ unsigned long long* cta_merge_sort(unsigned long long* bufA, unsigned long long* bufB, KeyOf&& key_of) {
  const int t = threadIdx.x, lane = t & 31;
  constexpr int P = NT * E, RUN0 = 32 * E;
  unsigned long long v[E];
#pragma unroll
  for (int s2 = 0; s2 < E; ++s2) v[s2] = key_of(t * E + s2);
  hybrid_bitonic<E, 32>(v, nullptr);   // warp-local: element index inside the warp = lane * E + slot
#pragma unroll
  for (int s2 = 0; s2 < E; ++s2) bufA[(t >> 5) * RUN0 + lane * E + s2] = v[s2];
  __syncthreads();
  unsigned long long* src = bufA;
  unsigned long long* dst = bufB;
#pragma unroll 1
  for (int L = RUN0; L < P; L <<= 1) {
    const int o = t * E;                 // first output slot of this thread
    const int pair0 = o & ~(2 * L - 1);  // start of the pair of runs it falls into
    const int d = o - pair0;             // diagonal inside the merged pair
    const unsigned long long* X = src + pair0;
    const unsigned long long* Y = src + pair0 + L;
    int lo = max(0, d - L), hi = min(d, L);
    while (lo < hi) {                    // smallest a with X[a] >= Y[d - 1 - a]  (ties: X first, the keys of real points are unique)
      const int mid = (lo + hi) >> 1;
      if (X[mid] <= Y[d - 1 - mid]) lo = mid + 1; else hi = mid;
    }
    int a = lo, b = d - lo;
    unsigned long long xa = a < L ? X[a] : ~0ull, yb = b < L ? Y[b] : ~0ull;
#pragma unroll
    for (int s2 = 0; s2 < E; ++s2) {
      const bool take_x = b >= L || (a < L && xa <= yb);
      dst[o + s2] = take_x ? xa : yb;
      if (take_x) { ++a; xa = a < L ? X[a] : ~0ull; } else { ++b; yb = b < L ? Y[b] : ~0ull; }
    }
    __syncthreads();
    unsigned long long* tmp = src; src = dst; dst = tmp;
  }
  return src;
}

// gap bit i = |p[i+1]-p[i]|^2 > 0.05 (float expression compared with the double literal, :324)
__device__ __forceinline__ unsigned bits5(const unsigned* m, int from) {  // 5 bits starting at bit `from`
  unsigned long long two = (unsigned long long)m[from >> 5] | ((unsigned long long)m[(from >> 5) + 1] << 32);
  return (unsigned)(two >> (from & 31)) & 31u;
}
__device__ __forceinline__ void suppress_range(const unsigned* gap, int ind, int& lo, int& hi) {
  unsigned fw = bits5(gap, ind);           // gaps (ind,ind+1) .. (ind+4,ind+5)
  int f = fw ? (__ffs(fw) - 1) : 5;
  unsigned bw = bits5(gap, ind - 5);       // gaps (ind-5,ind-4) .. (ind-1,ind) ; walk down from bit 4
  int b = bw ? (4 - (31 - __clz(bw))) : 5;
  lo = ind - b; hi = ind + f;
}
__device__ __forceinline__ void set_bits(unsigned* m, int lo, int hi) {  // single warp, called by one lane
  for (int w = lo >> 5; w <= (hi >> 5); ++w) {
    int a = max(lo, w << 5) & 31, b = min(hi, (w << 5) + 31) & 31;
    unsigned mask = (b == 31 ? 0xffffffffu : ((1u << (b + 1)) - 1u)) & ~((1u << a) - 1u);
    m[w] |= mask;
  }
}

}  // namespace

// One sixth of a ring (:282-398 minus the sort): positions [sp, ep], lane owns positions sp + 32 s + lane.
// spill_in : bit k set = position sp + k was marked in cloudNeighborPicked by the previous segment's picks (k < 5).
// Results (warp-uniform): `less` = positions picked in the sharp walk in pick order (the first two are the sharp
// points), `flat` = positions of the flat walk, spill_out = marks this segment leaves on positions ep+1 .. ep+5.
template <int NS>
__device__ __forceinline__ void pick_segment(const float* curv, const unsigned char* fb, int sp, int ep, unsigned spill_in,
                                             unsigned short* less, int& n_less, unsigned short* flat, int& n_flat,
                                             unsigned& spill_out, bool dbg_seg) {
  const int lane = threadIdx.x & 31;
  const bool dbg_me = dbg_seg && lane == 0;
  if (dbg_me) g_dbg_pick[0] = clock64();
  float c[NS];
  unsigned valid = 0, pk = 0;   // bit s: slot s is inside the segment / is marked in cloudNeighborPicked
#pragma unroll
  for (int s2 = 0; s2 < NS; ++s2) {
    const int p = sp + s2 * 32 + lane;
    c[s2] = 0.f;
    if (p <= ep) { c[s2] = curv[p]; valid |= 1u << s2; }
  }
  if (lane < 5 && sp + lane <= ep) pk |= (spill_in >> lane) & 1u;   // slot 0 of lanes 0..4
  spill_out = 0;
  // marks the slot of this lane that falls inside [lo, hi] (at most one: the range is <= 11 long) ; records the spill
  auto mark = [&](int lo, int hi) {
    const int t = (lane - (lo - sp)) & 31;
    const int p = lo + t;
    if (p <= hi && p >= sp && p <= ep) pk |= 1u << ((p - sp) >> 5);
    if (hi > ep) spill_out |= ((1u << (hi - ep)) - 1u) & ~((lo > ep + 1) ? ((1u << (lo - ep - 1)) - 1u) : 0u);
  };
  n_less = 0; n_flat = 0;
  if (dbg_me) g_dbg_pick[1] = clock64();
  // ---- largest curvature first (:291-344): eligible = !picked && c > 0.1 ; ties -> larger index (top of the sorted run)
  // The local scan is written as independent operations (a max tree, then "highest slot equal to the maximum" from a bit
  // mask) instead of a 12-deep dependent compare / select chain: the warp runs alone on its scheduler, so instruction-level
  // parallelism is the only latency hiding there is.  An eligible curvature is > 0.1, i.e. its bit pattern is non-zero,
  // so a warp maximum of 0 means "nobody eligible" and no separate vote is needed.  (A 64-bit shuffle butterfly instead of
  // the two REDUX was measured: 2.2x slower.)
  unsigned el = 0;
#pragma unroll
  for (int s2 = 0; s2 < NS; ++s2) if ((double)c[s2] > 0.1) el |= 1u << s2;
  el &= valid;
  unsigned cb[NS];
#pragma unroll
  for (int s2 = 0; s2 < NS; ++s2) cb[s2] = __float_as_uint(c[s2]);
  for (;;) {
    const unsigned e = el & ~pk;
    unsigned kk[NS];
#pragma unroll
    for (int s2 = 0; s2 < NS; ++s2) kk[s2] = ((e >> s2) & 1u) ? cb[s2] : 0u;
    unsigned t[NS];
#pragma unroll
    for (int s2 = 0; s2 < NS; ++s2) t[s2] = kk[s2];
#pragma unroll
    for (int w2 = 1; w2 < NS; w2 <<= 1) {
#pragma unroll
      for (int s2 = 0; s2 + w2 < NS; s2 += 2 * w2) t[s2] = max(t[s2], t[s2 + w2]);
    }
    const unsigned bb = t[0];
    const unsigned mx = __reduce_max_sync(0xffffffffu, bb);
    if (mx == 0u) break;
    unsigned mm = 0;
#pragma unroll
    for (int s2 = 0; s2 < NS; ++s2) mm |= (kk[s2] == mx) ? (1u << s2) : 0u;
    const int cand = mm ? (sp + (31 - __clz(mm)) * 32 + lane) : -1;   // later slot = larger position wins a tie inside a lane
    const int win = __reduce_max_sync(0xffffffffu, cand);
    if (n_less >= 20) break;          // the 21st eligible point ends the walk unpicked (:312-315)
    const unsigned char r = fb[win];
    if (lane == 0) less[n_less] = (unsigned short)win;
    ++n_less;
    mark(win - (r >> 4), win + (r & 15));
  }
  if (dbg_me) g_dbg_pick[2] = clock64();
  // ---- smallest curvature first (:346-390): eligible = !picked && c < 0.1 ; ties -> smaller index ; 4th pick not marked
  el = 0;
#pragma unroll
  for (int s2 = 0; s2 < NS; ++s2) if ((double)c[s2] < 0.1) el |= 1u << s2;
  el &= valid;
  for (;;) {
    const unsigned e = el & ~pk;
    unsigned kk[NS];
#pragma unroll
    for (int s2 = 0; s2 < NS; ++s2) kk[s2] = ((e >> s2) & 1u) ? cb[s2] : 0xffffffffu;   // curvatures are finite: their bits are below 0x7f800000
    unsigned t[NS];
#pragma unroll
    for (int s2 = 0; s2 < NS; ++s2) t[s2] = kk[s2];
#pragma unroll
    for (int w2 = 1; w2 < NS; w2 <<= 1) {
#pragma unroll
      for (int s2 = 0; s2 + w2 < NS; s2 += 2 * w2) t[s2] = min(t[s2], t[s2 + w2]);
    }
    const unsigned bb = t[0];
    const unsigned mn = __reduce_min_sync(0xffffffffu, bb);
    if (mn == 0xffffffffu) break;
    unsigned mm = 0;
#pragma unroll
    for (int s2 = 0; s2 < NS; ++s2) mm |= (kk[s2] == mn) ? (1u << s2) : 0u;
    const int cand = mm ? (sp + (__ffs(mm) - 1) * 32 + lane) : 0x7fffffff;   // earlier slot = smaller position wins a tie inside a lane
    const int win = __reduce_min_sync(0xffffffffu, cand);
    if (lane == 0) flat[n_flat] = (unsigned short)win;
    ++n_flat;
    if (n_flat >= 4) break;
    const unsigned char r = fb[win];
    mark(win - (r >> 4), win + (r & 15));
  }
  if (dbg_me) { g_dbg_pick[3] = clock64(); g_dbg_pick[4] = n_less; g_dbg_pick[5] = n_flat; }
  __syncwarp();
}

__device__ long long g_dbg_cycles[65 * 8];   // per-ring phase time stamps (clock64) of the last k_ring_features launch

// dynamic shared memory layout (bytes), maxr = ring capacity of the context (multiple of 32, <= ALOAM_MAX_RING), P = sort width
// (next power of two >= maxr, >= 1024):  pts 16*maxr | keys 8*P | curv 4*maxr | label maxr | gap 4*(maxr/32+2) | picked same | fb maxr
// The smaller the ring capacity the more CTAs are resident per SM (2048: 65 KB -> 3 per SM; 4096: 131 KB -> 1 per SM),
// which is what a batch of trajectories needs.
__host__ __device__ inline int sort_width(int maxr) { int p = 1024; while (p < maxr) p <<= 1; return p; }
// merge = the 512-thread kernel, which sorts by merging and needs a second key buffer (placed after everything else)
size_t ring_features_smem_bytes(int maxr, bool merge) {
  return (size_t)maxr * (16 + 4 + 1 + 1) + (size_t)sort_width(maxr) * 8 * (merge ? 2 : 1) + 2 * 4 * (maxr / 32 + 2) + 64;
}

// ---- thread-block-cluster helpers of the paired kernel (raw PTX: the barrier is used split, arrive now / wait later)
__device__ __forceinline__ unsigned cluster_cta_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void st_dsmem_s8(void* local, unsigned rank, int v) {   // the same shared-memory offset in CTA `rank` of the cluster
  const unsigned a = (unsigned)__cvta_generic_to_shared(local);
  unsigned ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a), "r"(rank));
  asm volatile("st.shared::cluster.u8 [%0], %1;" ::"r"(ra), "r"(v) : "memory");
}

// RFT = threads of a ring CTA: six warps walk the segments, all of them load, sort and sum.
//   PAIR = false : one CTA does the whole ring (256 threads, two or three CTAs per SM): batches of trajectories, which fill the GPU.
//   PAIR = true  : a single trajectory, where the kernel is a latency chain on 64 of the GPU's SMs.  A ring is processed by a CLUSTER
//                  OF TWO CTAs on two SMs: rank 0 = curvature, greedy picks, labels, the three picked clouds ; rank 1 = the voxel
//                  sort of the ring, which is made INDEPENDENT of the picks: it sorts every in-range position by its absolute voxel
//                  coordinates (floor(z/leaf), floor(y/leaf), floor(x/leaf)) -- the same order as PCL's index relative to the
//                  bounding box of the candidates, because that index is lexicographic in (z, y, x) -- and removes the picked
//                  positions afterwards, using rank 0's labels, which rank 0 pushes into rank 1's shared memory (DSMEM stores).  The two halves overlap;
//                  the chain is max(picks, sort) + centroids instead of their sum.
template <int RFT, bool PAIR>
__device__ __forceinline__ void ring_features_body(const Batch<RingFeatArgs>& B, int n_scans, float leaf, int MAXR) {
  pdl_launch_dependents();   // the next kernel of the stream may become resident (it blocks in pdl_wait())
  const RingFeatArgs& A = B.a[blockIdx.y];   // blockIdx.x = ring (PAIR: 2 * ring + cluster rank), blockIdx.y = trajectory of the batch
  const Pt4* __restrict__ full = A.full;
  const int* __restrict__ ring_start = A.ring_start;
  Pt4* __restrict__ st_sharp = A.st_sharp;
  Pt4* __restrict__ st_less_sharp = A.st_less_sharp;
  Pt4* __restrict__ st_flat = A.st_flat;
  Pt4* __restrict__ st_less_flat = A.st_less_flat;
  int* __restrict__ st_counts = A.st_counts;
  float* __restrict__ dbg_curv = A.dbg_curv;
  int8_t* __restrict__ dbg_label = A.dbg_label;
  ScanScalars* __restrict__ sc = A.sc;
  extern __shared__ __align__(16) unsigned char smem[];
  const int PW = sort_width(MAXR);
  Pt4* pts = reinterpret_cast<Pt4*>(smem);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem + (size_t)MAXR * 16);
  float* curv = reinterpret_cast<float*>(smem + (size_t)MAXR * 16 + (size_t)PW * 8);
  signed char* label = reinterpret_cast<signed char*>(curv + MAXR);
  unsigned* gap = reinterpret_cast<unsigned*>(label + MAXR);
  unsigned* picked = gap + (MAXR / 32 + 2);
  unsigned char* fb = reinterpret_cast<unsigned char*>(picked + (MAXR / 32 + 2));   // [MAXR]
  unsigned long long* keys2 = reinterpret_cast<unsigned long long*>(smem + (((size_t)(fb + MAXR - smem) + 15) & ~(size_t)15));   // [PW], 512-thread kernel only
  __shared__ unsigned short s_less[6][20], s_flat[6][4];
  __shared__ int s_nl[6], s_nf[6];
  __shared__ unsigned s_spill[6], s_in[6];
  __shared__ int s_i[RFT / 32];
  __shared__ float s_red[6][RFT / 32];

  // role 0: the whole ring ; 1: the picks CTA of a pair ; 2: the voxel CTA of a pair
  const int role = PAIR ? (int)cluster_cta_rank() + 1 : 0;
  const int ring = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool stamp = g_dbg_stamp != 0;
  const bool dbg8 = stamp && ring == 8 && blockIdx.y == 0;
  const int g0 = ring_start[ring], nr = ring_start[ring + 1] - g0;
  int* counts = st_counts + ring * 4;
  if (nr > MAXR) {   // (both CTAs of a pair leave here, before any cluster barrier)
    if (tid == 0 && role != 2) { sc->error = ALOAM_ERR_RING_TOO_LARGE_DEV; counts[0] = counts[1] = counts[2] = counts[3] = 0; }
    return;
  }
  // scanStartInd = g0+5, scanEndInd = g0+nr-6 ; skip ring if end - start < 6 (:279)
  const int s_loc = 5, e_loc = nr - 6;
  for (int i = tid; i < nr; i += blockDim.x) {
    label[i] = 0;
    if (role != 2) { if (dbg_label) dbg_label[g0 + i] = 0; if (dbg_curv) dbg_curv[g0 + i] = 0.f; }
  }
  if (e_loc - s_loc < 6) {
    if (tid == 0 && role != 2) counts[0] = counts[1] = counts[2] = counts[3] = 0;
    return;
  }
  int P = 32;
  while (P < nr) P <<= 1;

  long long* dbg = g_dbg_cycles + (blockIdx.y == 0 ? ring : 64) * 8;   // lane 0 only; the other lanes write a dummy row
  if (stamp && tid == 0) dbg[role == 2 ? 7 : 0] = clock64();
  // The ring (nr x 16 bytes, up to 64 KB, contiguous in the ring-major cloud) is staged into shared memory by ONE TMA bulk copy
  // (cp.async.bulk, 1-D): a single thread arms an mbarrier with the byte count and issues the copy, the copy engine moves the
  // tile while the CTA clears its bit arrays, and everybody waits on the barrier's phase.  (Before: every thread looped over
  // LDG.128 + STS.128 pairs.)
  __shared__ __align__(8) unsigned long long s_bar;
  const unsigned bar = (unsigned)__cvta_generic_to_shared(&s_bar);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned bytes = (unsigned)nr * 16u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (unsigned)__cvta_generic_to_shared(pts)),
                 "l"(full + g0), "r"(bytes), "r"(bar)
                 : "memory");
  }
  for (int i = tid; i < MAXR / 32 + 2; i += blockDim.x) { gap[i] = 0; picked[i] = 0; }
  {
    unsigned done = 0;
    while (!done)
      asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(done) : "r"(bar) : "memory");
  }
  __syncthreads();
  // pair, barrier Z: the voxel CTA's label array is zeroed -- the picks CTA will PUSH the few non-zero labels into it
  if (role != 0) cluster_arrive();
  if (role == 2) cluster_wait();

  if (role != 2) {
  // curvature (:256-266) for local 5 .. nr-6, left-to-right float sums ; gap bits (whole warps iterate together)
  for (int base = warp * 32; base < nr; base += blockDim.x) {
    const int i = base + lane;
    float c = 0.f;
    bool g = false;
    if (i < nr) {
      if (i >= 5 && i < nr - 5) {
        float dx = pts[i - 5].x + pts[i - 4].x + pts[i - 3].x + pts[i - 2].x + pts[i - 1].x - 10 * pts[i].x + pts[i + 1].x + pts[i + 2].x + pts[i + 3].x + pts[i + 4].x + pts[i + 5].x;
        float dy = pts[i - 5].y + pts[i - 4].y + pts[i - 3].y + pts[i - 2].y + pts[i - 1].y - 10 * pts[i].y + pts[i + 1].y + pts[i + 2].y + pts[i + 3].y + pts[i + 4].y + pts[i + 5].y;
        float dz = pts[i - 5].z + pts[i - 4].z + pts[i - 3].z + pts[i - 2].z + pts[i - 1].z - 10 * pts[i].z + pts[i + 1].z + pts[i + 2].z + pts[i + 3].z + pts[i + 4].z + pts[i + 5].z;
        c = dx * dx + dy * dy + dz * dz;
      }
      curv[i] = c;
      if (dbg_curv) dbg_curv[g0 + i] = c;
      if (i + 1 < nr) {
        float dx = pts[i + 1].x - pts[i].x, dy = pts[i + 1].y - pts[i].y, dz = pts[i + 1].z - pts[i].z;
        g = (double)(dx * dx + dy * dy + dz * dz) > 0.05;
      }
    }
    unsigned bal = __ballot_sync(0xffffffffu, g);
    if (lane == 0) gap[base >> 5] = bal;
  }
  // suppression reach of every position (:319-342): fb = forward count | backward count << 4, from the gap bits
  const int span = e_loc - s_loc;
  __syncthreads();
  for (int i = tid; i < nr; i += blockDim.x) {
    unsigned char v = 0;
    if (i >= 5 && i < nr - 5) { int lo, hi; suppress_range(gap, i, lo, hi); v = (unsigned char)((hi - i) | ((i - lo) << 4)); }
    fb[i] = v;
  }
  __syncthreads();
  if (stamp && tid == 0) { dbg[1] = clock64(); dbg[2] = dbg[1]; }

  // greedy picks (:291-390).  std::sort + walk == repeatedly taking the arg-max (arg-min) of the still-eligible
  // points under the (curvature, index) order, so no sort is needed: one warp keeps a segment's curvatures in
  // registers (position sp + 32 s + lane in slot s) and performs <= 20 + 4 REDUX selections.
  // The six segments of a ring depend on each other only through the <= 5 marks a segment spills onto the start of
  // the next one (:319-330).  Six warps therefore process the six segments CONCURRENTLY assuming an empty spill;
  // a segment is re-run (in order) only if a position actually spilled onto it is one of its own picks -- removing a
  // point that never wins a selection cannot change any selection, so otherwise the speculative result is exact.
  auto run_segment = [&](int w, unsigned spill_in) {
    const int sp = s_loc + span * w / 6, ep = s_loc + span * (w + 1) / 6 - 1;
    int nl, nf; unsigned so;
    if (ep - sp + 1 <= 12 * 32) pick_segment<12>(curv, fb, sp, ep, spill_in, s_less[w], nl, s_flat[w], nf, so, dbg8 && w == 2);
    else pick_segment<24>(curv, fb, sp, ep, spill_in, s_less[w], nl, s_flat[w], nf, so, dbg8 && w == 2);
    if (lane == 0) { s_nl[w] = nl; s_nf[w] = nf; s_spill[w] = so; }
  };
  // Warps 1..6 walk the six segments.  NOT warp 0: it carries the thread that writes the debug stamps, so its REDUX go
  // through the divergent-warp path and a segment walk there is slower than on any other warp.
  if (warp >= 1 && warp <= 6) {
    if (dbg8 && lane == 0) g_dbg_pick[8 + 2 * (warp - 1)] = clock64();
    run_segment(warp - 1, 0u);
    if (dbg8 && lane == 0) g_dbg_pick[9 + 2 * (warp - 1)] = clock64();
  }
  if (tid < 6) s_in[tid] = 0u;   // the incoming spill every segment was walked with
  if (dbg8 && tid == 0) g_dbg_pick[6] = clock64();
  // Fixed-point rounds instead of a sequential sweep over the boundaries: every segment compares the spill its predecessor
  // CURRENTLY reports (S) with the one it was walked with (A) and walks again, all such segments in parallel, if the difference
  // can matter: a mark it assumed is not there (A & ~S), or a new mark sits on one of its own picks.  Otherwise its result is
  // also the result for S.  When a round changes nothing every segment is consistent with its predecessor, and segment 0
  // (no predecessor) is exact, so by induction all are; the lowest inconsistent segment becomes final in every round, hence
  // at most five rounds -- typically one, where the sequential sweep paid one walk per conflict.
  for (;;) {
    __syncthreads();
    bool need = false;
    unsigned S = 0u;
    if (warp >= 2 && warp <= 6) {
      const int w = warp - 1;
      S = s_spill[w - 1];
      const unsigned Ain = s_in[w];
      if (S != Ain) {
        const int sp = s_loc + span * w / 6;
        const int nl = s_nl[w], nf = s_nf[w];
        const unsigned fresh = S & ~Ain;
        bool hit = (Ain & ~S) != 0u;
        if (lane < nl) { const int k = (int)s_less[w][lane] - sp; hit = hit || (k < 5 && ((fresh >> k) & 1u)); }
        if (lane >= 24 && lane - 24 < nf) { const int k = (int)s_flat[w][lane - 24] - sp; hit = hit || (k < 5 && ((fresh >> k) & 1u)); }
        need = __any_sync(0xffffffffu, hit);
      }
    }
    if (!__syncthreads_or(need ? 1 : 0)) break;   // (also orders this round's reads of s_spill / s_less before the walks' writes)
    if (warp >= 2 && warp <= 6) {
      const int w = warp - 1;
      if (need) run_segment(w, S);
      if (lane == 0) s_in[w] = S;   // walked with S, or its result is the result for S as well
    }
  }
  if (dbg8 && tid == 0) g_dbg_pick[7] = clock64();
  // labels (:303,309,355) and ring-ordered outputs (ring, segment, pick order) from the per-segment lists
  if (role == 1) { __syncwarp(); cluster_wait(); }   // barrier Z (arrived at the start): the voxel CTA has zeroed its labels
  if (tid < 6 * 24) {
    const int w = tid / 24, i = tid % 24;
    int o_sh = 0, o_ls = 0, o_fl = 0;
    for (int v = 0; v < w; ++v) { o_sh += min(2, s_nl[v]); o_ls += s_nl[v]; o_fl += s_nf[v]; }
    if (i < s_nl[w]) {
      const int p = s_less[w][i];
      label[p] = i < 2 ? 2 : 1;
      if (role == 1) st_dsmem_s8(label + p, 1u, i < 2 ? 2 : 1);
      if (i < 2) st_sharp[ring * 12 + o_sh + i] = pts[p];
      st_less_sharp[ring * 120 + o_ls + i] = pts[p];
    }
    if (i >= 20 && i - 20 < s_nf[w]) {
      const int p = s_flat[w][i - 20];
      label[p] = -1;
      if (role == 1) st_dsmem_s8(label + p, 1u, -1);
      st_flat[ring * 24 + o_fl + (i - 20)] = pts[p];
    }
    if (tid == 0) {
      int a2 = 0, b2 = 0, c2 = 0;
      for (int v = 0; v < 6; ++v) { a2 += min(2, s_nl[v]); b2 += s_nl[v]; c2 += s_nf[v]; }
      counts[0] = a2; counts[1] = b2; counts[2] = c2;
    }
  }
  __syncthreads();
  if (role == 1) cluster_arrive();   // barrier A (release): the labels are final and pushed
  if (stamp && tid == 0) dbg[3] = clock64();
  if (dbg_label) for (int i = tid; i < nr; i += blockDim.x) dbg_label[g0 + i] = label[i];
  if (role == 1) {   // nothing of this CTA is read remotely: it leaves as soon as the barrier phase is complete
    __syncwarp();
    cluster_wait();
    return;
  }
  }   // role != 2

  // ---- less-flat candidates = positions [s_loc, e_loc-1] with label <= 0 (:392-398), voxel-filtered per ring (:401-407)
  // pcl::VoxelGrid::applyFilter: bounding box, voxel index, sort by (index, position), float centroid per voxel
  const float inv = 1.0f / leaf;  // inverse_leaf_size_ = Array4f::Ones() / leaf_size_
  // bounding box of the positions [s_loc, e_loc) accepted by `use`, reduced over the CTA (every thread gets the result)
  auto block_bbox = [&](auto&& use, float* mn, float* mx) {
    mn[0] = mn[1] = mn[2] = FLT_MAX; mx[0] = mx[1] = mx[2] = -FLT_MAX;
    for (int i = s_loc + tid; i < e_loc; i += blockDim.x) {
      if (use(i)) {
        mn[0] = fminf(mn[0], pts[i].x); mn[1] = fminf(mn[1], pts[i].y); mn[2] = fminf(mn[2], pts[i].z);
        mx[0] = fmaxf(mx[0], pts[i].x); mx[1] = fmaxf(mx[1], pts[i].y); mx[2] = fmaxf(mx[2], pts[i].z);
      }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], d));
        mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], d));
      }
      if (lane == 0) { s_red[a][warp] = mn[a]; s_red[3 + a][warp] = mx[a]; }
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      float lo = s_red[a][0], hi = s_red[3 + a][0];
      for (int w2 = 1; w2 < (int)(blockDim.x >> 5); ++w2) { lo = fminf(lo, s_red[a][w2]); hi = fmaxf(hi, s_red[3 + a][w2]); }
      mn[a] = lo; mx[a] = hi;
    }
    __syncthreads();   // s_red may be reused
  };
  auto grid_overflows = [&](const float* mn, const float* mx) {   // PCL: dx * dy * dz > INT_MAX -> the filter returns its input
    long long d[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) d[a] = (long long)((mx[a] - mn[a]) * inv) + 1;
    return mn[0] <= mx[0] && d[0] * d[1] * d[2] > (long long)INT_MAX;
  };
  if (P < 1024) P = 1024;
  auto sort_by = [&](auto&& key_of) {
    if (RFT == 512) {   // merge sort (two key buffers); the result may be in either buffer
      if (P == 1024) keys = cta_merge_sort<1024 / RFT, RFT>(keys, keys2, key_of);
      else if (P == 2048) keys = cta_merge_sort<2048 / RFT, RFT>(keys, keys2, key_of);
      else keys = cta_merge_sort<4096 / RFT, RFT>(keys, keys2, key_of);
    } else {            // batches: bitonic network in place (one key buffer: more CTAs per SM)
      if (P == 1024) cta_sort_keys<1024 / RFT, RFT>(keys, key_of);
      else if (P == 2048) cta_sort_keys<2048 / RFT, RFT>(keys, key_of);
      else cta_sort_keys<4096 / RFT, RFT>(keys, key_of);
    }
  };

  // The voxel CTA of a pair sorts BEFORE the labels exist.  Preconditions (CTA-uniform, from the bounding box of ALL in-range
  // positions, a superset of the candidates): every voxel coordinate fits 17 bits and the superset's grid does not overflow
  // (then the candidates' grid does not either).  Otherwise it falls back to the order of operations of the single CTA.
  bool presorted = false;
  if (role == 2) {
    float mn[3], mx[3];
    block_bbox([&](int) { return true; }, mn, mx);
    bool fits = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) fits = fits && floorf(mn[a] * inv) > -65536.f && floorf(mx[a] * inv) < 65536.f;
    presorted = fits && !grid_overflows(mn, mx);
    if (stamp && tid == 0) dbg[4] = clock64();
    if (presorted) {
      sort_by([&](int i) -> unsigned long long {
        if (!(i >= s_loc && i < e_loc)) return ~0ull;
        const unsigned long long ix = (unsigned long long)((int)floorf(pts[i].x * inv) + 65536);
        const unsigned long long iy = (unsigned long long)((int)floorf(pts[i].y * inv) + 65536);
        const unsigned long long iz = (unsigned long long)((int)floorf(pts[i].z * inv) + 65536);
        return ((((iz << 17) | iy) << 17 | ix) << 12) | (unsigned)i;   // 51 + 12 bits
      });
      if (stamp && tid == 0) dbg[5] = clock64();
    }
    // barrier A (acquire): rank 0's labels are final and sit in this CTA's label array
    __syncwarp();
    cluster_arrive();
    cluster_wait();
  }

  bool overflow = false;
  if (!presorted) {
    float mn[3], mx[3];
    block_bbox([&](int i) { return label[i] <= 0; }, mn, mx);
    int min_b[3], div_b[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      min_b[a] = (int)floorf(mn[a] * inv);
      div_b[a] = (int)floorf(mx[a] * inv) - min_b[a] + 1;
    }
    overflow = grid_overflows(mn, mx);
    if (stamp && tid == 0) dbg[4] = clock64();
    // keys: [voxel idx 32b | local position 12b], non-candidates last ; sorted by the whole CTA
    // (overflow case: idx = 0 everywhere => position order, i.e. output = input, PCL's early return)
    sort_by([&](int i) -> unsigned long long {
      if (!(i >= s_loc && i < e_loc && label[i] <= 0)) return ~0ull;
      unsigned idx = 0;
      if (!overflow) {
        const int i0 = (int)(floorf(pts[i].x * inv) - (float)min_b[0]);
        const int i1 = (int)(floorf(pts[i].y * inv) - (float)min_b[1]);
        const int i2 = (int)(floorf(pts[i].z * inv) - (float)min_b[2]);
        idx = (unsigned)(i0 + i1 * div_b[0] + i2 * div_b[0] * div_b[1]);
      }
      return ((unsigned long long)idx << 12) | (unsigned)i;
    });
    if (stamp && tid == 0) dbg[5] = clock64();
  }

  // A sorted slot is a candidate unless the presorted order still contains the picked positions ; a candidate is the head of its
  // voxel if no candidate precedes it in the voxel's run (picked positions are few, so the walk back is short).
  auto is_cand = [&](unsigned long long key) { return !presorted || label[(int)(key & 0xfffu)] <= 0; };
  auto is_head = [&](int k, unsigned long long key) {
    if (!is_cand(key)) return false;
    if (overflow) return true;
    for (int k2 = k - 1; k2 >= 0; --k2) {
      const unsigned long long kp = keys[k2];
      if ((kp >> 12) != (key >> 12)) break;
      if (is_cand(kp)) return false;
    }
    return true;
  };
  // head flags -> output slots ; each thread owns E consecutive sorted slots
  const int E = P / (int)blockDim.x > 0 ? P / (int)blockDim.x : 1;
  const int k0 = tid * E;
  unsigned head_bits = 0;   // E <= 16
  for (int k = k0; k < k0 + E && k < P; ++k) {
    const unsigned long long key = keys[k];
    if (key == ~0ull) break;
    if (is_head(k, key)) head_bits |= 1u << (k - k0);
  }
  const int heads = __popc(head_bits);
  // block exclusive scan of `heads`
  int incl = heads;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) s_i[warp] = incl;
  __syncthreads();
  int wbase = 0, total = 0;
  for (int w2 = 0; w2 < (int)(blockDim.x >> 5); ++w2) { if (w2 < warp) wbase += s_i[w2]; total += s_i[w2]; }
  int slot = wbase + incl - heads;
  Pt4* o_lf = st_less_flat + (size_t)ring * MAXR;
  // the heads' sorted positions, compacted: afterwards ONE thread per voxel sums its run (a thread that owned several
  // single-point voxels and one long run used to serialise them all)
  int* head_pos = reinterpret_cast<int*>(curv);   // the curvatures are not needed any more ; #voxels <= #points <= MAXR
  for (unsigned hb = head_bits; hb; hb &= hb - 1) head_pos[slot++] = k0 + __ffs(hb) - 1;
  __syncthreads();
  for (int h = tid; h < total; h += blockDim.x) {
    const int k = head_pos[h];
    const unsigned long long idx = keys[k] >> 12;
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
    int cnt = 0;
    for (int k2 = k; k2 < P; ++k2) {  // float accumulation in sorted order, then divide (pcl::CentroidPoint)
      const unsigned long long key2 = keys[k2];
      if (key2 == ~0ull || (!overflow && (key2 >> 12) != idx) || (overflow && k2 > k)) break;
      if (!is_cand(key2)) continue;
      const Pt4 p = pts[(int)(key2 & 0xfffu)];
      sx += p.x; sy += p.y; sz += p.z; si += p.i;
      ++cnt;
    }
    const float nf = (float)cnt;
    Pt4 o; o.x = sx / nf; o.y = sy / nf; o.z = sz / nf; o.i = si / nf;
    o_lf[h] = o;
  }
  if (tid == 0) { counts[3] = total; if (stamp) dbg[6] = clock64(); }
}

// grid (2 * rings, 1), clusters of two CTAs
__global__ void __launch_bounds__(512) k_ring_features(const __grid_constant__ Batch<RingFeatArgs> B, int n_scans, float leaf, int max_ring) {
  ring_features_body<512, true>(B, n_scans, leaf, max_ring);
}
__global__ void __launch_bounds__(256) k_ring_features_batch(const __grid_constant__ Batch<RingFeatArgs> B, int n_scans, float leaf, int max_ring) {
  ring_features_body<256, false>(B, n_scans, leaf, max_ring);
}

void features_debug_enable(int on) { cudaMemcpyToSymbol(g_dbg_stamp, &on, sizeof(int)); }
void features_debug_cycles(long long* host64x8) {
  cudaMemcpyFromSymbol(host64x8, g_dbg_cycles, sizeof(long long) * 64 * 8);
  cudaMemcpyFromSymbol(host64x8 + 64 * 8, g_dbg_pick, sizeof(long long) * 20);   // the buffer of the caller holds 65 rows
}

// ---------------------------------------------------------------------------------------------------------------
// ring-ordered concatenation of the staged per-ring outputs ; also ring_start tables of the two "less" clouds
__global__ void __launch_bounds__(128) k_compact(const __grid_constant__ Batch<CompactArgs> B, int n_scans, int MAXR) {
  pdl_launch_dependents();
  pdl_wait();   // launched with a programmatic dependency on the previous kernel of the stream
  const CompactArgs& A = B.a[blockIdx.y];
  const Pt4* __restrict__ st_sharp = A.st_sharp;
  const Pt4* __restrict__ st_less_sharp = A.st_less_sharp;
  const Pt4* __restrict__ st_flat = A.st_flat;
  const Pt4* __restrict__ st_less_flat = A.st_less_flat;
  const int* __restrict__ st_counts = A.st_counts;
  Pt4* __restrict__ sharp = A.sharp;
  Pt4* __restrict__ less_sharp = A.less_sharp;
  Pt4* __restrict__ flat = A.flat;
  Pt4* __restrict__ less_flat = A.less_flat;
  int* __restrict__ counts = A.counts;
  int* __restrict__ rs_less_sharp = A.rs_ls;
  int* __restrict__ rs_less_flat = A.rs_lf;
  __shared__ int s_off[4];
  const int ring = blockIdx.x, tid = threadIdx.x;
  if (tid < 4) {
    int off = 0;
    for (int r = 0; r < ring; ++r) off += st_counts[r * 4 + tid];
    s_off[tid] = off;
    if (tid == 1) rs_less_sharp[ring] = off;
    if (tid == 3) rs_less_flat[ring] = off;
    if (ring == n_scans - 1) {
      int tot = off + st_counts[ring * 4 + tid];
      counts[tid] = tot;
      if (tid == 1) for (int r = n_scans; r <= 64; ++r) rs_less_sharp[r] = tot;
      if (tid == 3) for (int r = n_scans; r <= 64; ++r) rs_less_flat[r] = tot;
    }
  }
  __syncthreads();
  const int c0 = st_counts[ring * 4], c1 = st_counts[ring * 4 + 1], c2 = st_counts[ring * 4 + 2], c3 = st_counts[ring * 4 + 3];
  for (int i = tid; i < c0; i += blockDim.x) sharp[s_off[0] + i] = st_sharp[ring * 12 + i];
  for (int i = tid; i < c1; i += blockDim.x) less_sharp[s_off[1] + i] = st_less_sharp[ring * 120 + i];
  for (int i = tid; i < c2; i += blockDim.x) flat[s_off[2] + i] = st_flat[ring * 24 + i];
  for (int i = tid; i < c3; i += blockDim.x) less_flat[s_off[3] + i] = st_less_flat[(size_t)ring * MAXR + i];
}

}  // namespace aloam
