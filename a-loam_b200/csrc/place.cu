// Place recognition (include/aloam_b200.h: aloam_set_place, aloam_place_*): the Scan Context descriptor of a scan, keyframes and
// loop candidates of mapping lanes inside the mapped stream calls, and brute-force queries against a database of keyframe records.
//   * k_place_gate: one CTA per record of a mapping frame -- the keyframe gate on the row's refined map pose (thread 0), then the
//     descriptor of the row's less-sharp / less-flat clouds (shared-memory atomicMax over order-preserving keys, so the maximum does
//     not depend on point order), its column norms and the record, appended to the lane's table.  The row's keyframe index is the
//     query index the next two launches read: a row that is not a keyframe makes their CTAs leave at once.
//   * k_place_dist: D and shift of one (query, keyframe) pair per 64 threads, thread s the shift s: the definition's double sums in
//     its order, one IEEE operation at a time.  k_place_describe is the gate's descriptor alone (aloam_place_describe).
//   * k_place_best: the k best keyframes per query by (D, index), k rounds of a block-wide minimum above the last one taken.
//   * k_place_load: checks the records of a database and computes their column norms (aloam_place_db_load).
#include "ctx.h"
#include "libm_atan.cuh"

namespace {
constexpr int kRings = ALOAM_PLACE_RINGS, kSectors = ALOAM_PLACE_SECTORS, kBins = kRings * kSectors;
constexpr int kRec = ALOAM_PLACE_RECORD_BYTES, kDescAt = 80;
constexpr int kMaxKeyframes = 65536, kMaxDb = 1 << 20;
constexpr long long kMaxPairs = 1LL << 24;   // (query, keyframe) pairs of one k_place_dist launch
constexpr int kDescThreads = 512;
constexpr int kDistPairs = 4;                // keyframes per k_place_dist CTA, 64 threads each
constexpr int kBestThreads = 512;
static_assert(kRec == kDescAt + 4 * kBins, "record layout");
}  // namespace

struct aloam::Place {
  aloam_place_opts opt = {80.f, 2.f, 0.0, 0, 1};
  int cap = 0;                                  // keyframes per lane the tables take (opt.max_keyframes)
  int alloc = 0;                                // keyframes per lane the tables have room for: the lanes' stride
  BufGroup tables;                              // d_rec, d_norm: empty while recording has never been on
  char* d_rec = nullptr;                        // [n_lanes][alloc] records
  double* d_norm = nullptr;                     // [n_lanes][alloc][60]
  int* d_count = nullptr;                       // [n_lanes]
  int upper[ALOAM_MAX_BATCH] = {};              // host bound on each lane's count (the mapped rows since its table was cleared)
  aloam_place_row* d_rows = nullptr;            // [kMaxStreamScans], and its pinned copy
  aloam_place_row* h_rows = nullptr;
  BufGroup db;                                  // the database: M records and their norms
  char* d_db = nullptr;
  double* d_db_norm = nullptr;
  int db_n = 0;
  BufGroup describe;                            // aloam_place_describe: the two uploaded clouds, and the descriptor
  Pt4* d_cloud[2] = {};
  float* d_desc = nullptr;
  BufGroup query;                               // aloam_place_query: the queries and the matches
  float* d_q = nullptr; long long q_cap = 0;
  aloam_place_match* d_match = nullptr; long long match_cap = 0;
  BufGroup pairs;                               // the pairs' D and shift, of the loop query and the database query
  double* d_dist = nullptr; int* d_shift = nullptr; long long pair_cap = 0;
  int* d_err = nullptr;
};

namespace {

// one query set of k_place_dist / k_place_best: query descriptor q (1200 floats) against keyframes 0 .. n-1 of (rec, norm).  In the
// stream form the query is the keyframe row->keyframe of the same table, against its keyframes 0 .. row->keyframe - 1 - exclude.
struct PlaceSet {
  const float* q;
  const char* rec;
  const double* norm;
  int n;
  aloam_place_row* row;   // stream form (q and n come from it), else null
};
struct PlaceSets {
  Batch<PlaceSet> s;      // stream form: set y = s.a[y]
  const float* q;         // database form: set y queries q + 1200 y against (rec, norm, n)
  const char* rec;
  const double* norm;
  int n, exclude;
  bool stream;
  double* dist;           // [set][stride]: D and shift of every pair
  int* shift;
  long long stride;
};
__device__ __forceinline__ PlaceSet place_set(const PlaceSets& S, int y) {
  if (!S.stream) return PlaceSet{S.q + (size_t)y * kBins, S.rec, S.norm, S.n, nullptr};
  PlaceSet p = S.s.a[y];
  const int qi = p.row->keyframe;
  if (qi < 0) { p.n = 0; return p; }
  p.q = reinterpret_cast<const float*>(p.rec + (size_t)qi * kRec + kDescAt);
  p.n = max(0, qi - S.exclude);
  return p;
}

// float -> unsigned key in the total order of IEEE bit patterns (-0 < +0); key 0 marks an empty bin
__device__ __forceinline__ unsigned ord_key(float v) {
  const unsigned b = __float_as_uint(v);
  return b & 0x80000000u ? ~b : b | 0x80000000u;
}
__device__ __forceinline__ float key_value(unsigned k) {
  if (k == 0u) return 0.f;
  return __uint_as_float(k & 0x80000000u ? k & 0x7fffffffu : ~k);
}
__device__ __forceinline__ void bin_point(const Pt4& p, float max_range, float z_offset, unsigned* key) {
  const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)));
  if (!(r < max_range)) return;
  const int ring = min(kRings - 1, (int)__fdiv_rn(__fmul_rn(r, 20.0f), max_range));
  float a = libm::atan2f(p.y, p.x);
  if (a < 0.f) a = __fadd_rn(a, 6.28318548f);
  const int sector = min(kSectors - 1, (int)__fdiv_rn(__fmul_rn(a, 60.0f), 6.28318548f));
  atomicMax(&key[ring * kSectors + sector], ord_key(__fadd_rn(p.z, z_offset)));
}
// the block's descriptor of clouds a (na points) and b (nb points) into desc, and its column norms into norm (may be null)
__device__ void describe_block(const Pt4* a, int na, const Pt4* b, int nb, float max_range, float z_offset, unsigned* key, float* desc,
                               double* norm) {
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) key[i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < na + nb; i += blockDim.x) bin_point(i < na ? a[i] : b[i - na], max_range, z_offset, key);
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) desc[i] = key_value(key[i]);
  if (norm && threadIdx.x < kSectors) {
    const int c = threadIdx.x;
    double s = 0.0;
    for (int r = 0; r < kRings; ++r) { const double v = key_value(key[r * kSectors + c]); s = __dadd_rn(s, __dmul_rn(v, v)); }
    norm[c] = __dsqrt_rn(s);
  }
}

// ---- k_place_gate: one record of a mapping frame
struct PlaceGate {
  const Pt4* corner; const int* nc; const Pt4* surf; const int* ns;
  const double* pose;    // the row's refined map pose
  char* rec; double* norm; int* count;   // the lane's table
  aloam_place_row* row;
  int scan, lane, start;
};
__global__ void __launch_bounds__(kDescThreads) k_place_gate(const __grid_constant__ Batch<PlaceGate> B, int cap, float max_range, float z_offset,
                                                             double gap2) {
  const PlaceGate& g = B.a[blockIdx.x];
  __shared__ unsigned key[kBins];
  __shared__ int s_idx;
  if (threadIdx.x == 0) {
    const int n = g.start ? 0 : *g.count;
    bool kf = n == 0;
    if (!kf) {
      const double* last = reinterpret_cast<const double*>(g.rec + (size_t)(n - 1) * kRec);
      const double dx = __dsub_rn(g.pose[4], last[4]), dy = __dsub_rn(g.pose[5], last[5]), dz = __dsub_rn(g.pose[6], last[6]);
      kf = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) >= gap2;
    }
    const int idx = kf && n < cap ? n : -1;
    *g.row = aloam_place_row{idx, -1, -1, kf && n >= cap ? 1 : 0, -1.0};
    *g.count = idx >= 0 ? idx + 1 : n;
    s_idx = idx;
  }
  __syncthreads();
  const int idx = s_idx;
  if (idx < 0) return;
  char* r = g.rec + (size_t)idx * kRec;
  describe_block(g.corner, *g.nc, g.surf, *g.ns, max_range, z_offset, key, reinterpret_cast<float*>(r + kDescAt), g.norm + (size_t)idx * kSectors);
  if (threadIdx.x < 7) reinterpret_cast<double*>(r)[threadIdx.x] = g.pose[threadIdx.x];
  if (threadIdx.x == 7) {
    int* h = reinterpret_cast<int*>(r + 56);
    h[0] = g.scan; h[1] = g.lane;
    reinterpret_cast<float*>(r + 64)[0] = max_range; reinterpret_cast<float*>(r + 64)[1] = z_offset;
    h[4] = 0; h[5] = 0;
  }
}

__global__ void __launch_bounds__(kDescThreads) k_place_describe(const Pt4* a, int na, const Pt4* b, int nb, float max_range, float z_offset, float* desc) {
  __shared__ unsigned key[kBins];
  describe_block(a, na, b, nb, max_range, z_offset, key, desc, nullptr);
}

// ---- k_place_dist: grid (ceil(n_upper / kDistPairs), sets), kDistPairs x 64 threads, dynamic shared memory place_dist_smem()
constexpr size_t place_dist_smem() { return sizeof(double) * ((1 + kDistPairs) * (kBins + kSectors) + kDistPairs * 64); }
__global__ void __launch_bounds__(kDistPairs * 64) k_place_dist(const __grid_constant__ PlaceSets S) {
  const PlaceSet P = place_set(S, blockIdx.y);
  const int j0 = blockIdx.x * kDistPairs;
  if (j0 >= P.n) return;   // block-uniform
  extern __shared__ double sm[];
  double* qd = sm;                                  // [1200]
  double* qn = qd + kBins;                          // [60]
  double* kd = qn + kSectors;                       // [kDistPairs][1200]
  double* kn = kd + kDistPairs * kBins;             // [kDistPairs][60]
  double* ds = kn + kDistPairs * kSectors;          // [kDistPairs][64]
  const int np = min(kDistPairs, P.n - j0);
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) qd[i] = (double)P.q[i];
  for (int i = threadIdx.x; i < np * kBins; i += blockDim.x) {
    const int p = i / kBins, b = i - p * kBins;
    kd[i] = (double)reinterpret_cast<const float*>(P.rec + (size_t)(j0 + p) * kRec + kDescAt)[b];
  }
  for (int i = threadIdx.x; i < np * kSectors; i += blockDim.x) kn[i] = P.norm[(size_t)j0 * kSectors + i];
  __syncthreads();
  if (threadIdx.x < kSectors) {
    const int c = threadIdx.x;
    double s = 0.0;
    for (int r = 0; r < kRings; ++r) s = __dadd_rn(s, __dmul_rn(qd[r * kSectors + c], qd[r * kSectors + c]));
    qn[c] = __dsqrt_rn(s);
  }
  __syncthreads();
  const int p = threadIdx.x >> 6, s = threadIdx.x & 63;
  if (p < np && s < kSectors) {
    const double* d = kd + p * kBins;
    const double* dn = kn + p * kSectors;
    double sim = 0.0;
    int cnt = 0;
    for (int c = 0; c < kSectors; ++c) {
      int c2 = c + s;
      if (c2 >= kSectors) c2 -= kSectors;
      const double a = qn[c], b = dn[c2];
      if (a == 0.0 || b == 0.0) continue;
      double dot = 0.0;
#pragma unroll
      for (int r = 0; r < kRings; ++r) dot = __dadd_rn(dot, __dmul_rn(qd[r * kSectors + c], d[r * kSectors + c2]));
      sim = __dadd_rn(sim, __ddiv_rn(dot, __dmul_rn(a, b)));
      ++cnt;
    }
    ds[p * 64 + s] = cnt ? __dsub_rn(1.0, __ddiv_rn(sim, (double)cnt)) : 1.0;
  }
  __syncthreads();
  if (p < np && s == 0) {
    double best = ds[p * 64];
    int bs = 0;
    for (int k = 1; k < kSectors; ++k) if (ds[p * 64 + k] < best) { best = ds[p * 64 + k]; bs = k; }
    const size_t o = (size_t)blockIdx.y * S.stride + j0 + p;
    S.dist[o] = best;
    S.shift[o] = bs;
  }
}

// ---- k_place_best: grid (sets), kBestThreads threads.  Rank key (D, index): D's bits in total order, then the index.
__device__ __forceinline__ unsigned long long ord_key64(double v) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return b & 0x8000000000000000ull ? ~b : b | 0x8000000000000000ull;
}
__device__ __forceinline__ bool key_less(unsigned long long ka, int ja, unsigned long long kb, int jb) { return ka < kb || (ka == kb && ja < jb); }
__global__ void __launch_bounds__(kBestThreads) k_place_best(const __grid_constant__ PlaceSets S, int k, aloam_place_match* out) {
  const PlaceSet P = place_set(S, blockIdx.x);
  if (P.n <= 0) return;   // block-uniform; a stream row keeps the -1 fields k_place_gate wrote
  const double* dist = S.dist + (size_t)blockIdx.x * S.stride;
  const int* shift = S.shift + (size_t)blockIdx.x * S.stride;
  __shared__ unsigned long long wk[kBestThreads / 32];
  __shared__ int wj[kBestThreads / 32];
  unsigned long long pk = 0; int pj = -1;   // the last key taken (none yet)
  for (int r = 0; r < k; ++r) {
    unsigned long long bk = ~0ull; int bj = -1;
    for (int j = threadIdx.x; j < P.n; j += blockDim.x) {
      const unsigned long long kj = ord_key64(dist[j]);
      if (pj >= 0 && !key_less(pk, pj, kj, j)) continue;
      if (bj < 0 || key_less(kj, j, bk, bj)) { bk = kj; bj = j; }
    }
    for (int o = 16; o; o >>= 1) {
      const unsigned long long ok = __shfl_down_sync(0xffffffffu, bk, o);
      const int oj = __shfl_down_sync(0xffffffffu, bj, o);
      if (oj >= 0 && (bj < 0 || key_less(ok, oj, bk, bj))) { bk = ok; bj = oj; }
    }
    if (lane_id() == 0) { wk[threadIdx.x >> 5] = bk; wj[threadIdx.x >> 5] = bj; }
    __syncthreads();
    bk = wk[0]; bj = wj[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (wj[w] >= 0 && (bj < 0 || key_less(wk[w], wj[w], bk, bj))) { bk = wk[w]; bj = wj[w]; }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (P.row) { P.row->loop = bj; P.row->shift = shift[bj]; P.row->distance = dist[bj]; }
      else out[(size_t)blockIdx.x * k + r] = aloam_place_match{bj, shift[bj], dist[bj]};
    }
    pk = bk; pj = bj;
  }
}

// ---- k_place_load: grid (records), 64 threads: err bit 0 = a record is refused; its norms into norm
__global__ void k_place_load(const char* rec, double* norm, unsigned range_bits, unsigned offset_bits, int* err) {
  const char* r = rec + (size_t)blockIdx.x * kRec;
  const float* d = reinterpret_cast<const float*>(r + kDescAt);
  bool bad = false;
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) bad |= !isfinite(d[i]);
  if (threadIdx.x < 7) bad |= !isfinite(reinterpret_cast<const double*>(r)[threadIdx.x]);
  if (threadIdx.x == 7) bad |= reinterpret_cast<const unsigned*>(r + 64)[0] != range_bits || reinterpret_cast<const unsigned*>(r + 64)[1] != offset_bits;
  if (bad) atomicOr(err, 1);
  if (threadIdx.x < kSectors) {
    double s = 0.0;
    for (int k = 0; k < kRings; ++k) { const double v = d[k * kSectors + threadIdx.x]; s = __dadd_rn(s, __dmul_rn(v, v)); }
    norm[(size_t)blockIdx.x * kSectors + threadIdx.x] = __dsqrt_rn(s);
  }
}

unsigned bits_of(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

// the context's Place with its error word, keyframe counts and row tables, created on first use and released by aloam_destroy
int place_ensure(aloam_ctx* c) {
  if (c->place) return ALOAM_OK;
  if (cudaFuncSetAttribute(k_place_dist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)place_dist_smem()) != cudaSuccess) {
    cudaGetLastError(); return ALOAM_ERR_CUDA;
  }
  Place* P = new (std::nothrow) Place();
  if (!P) return ALOAM_ERR_CUDA;
  BufGroup g;
  if (!g.dev(&P->d_err, 1) || !g.dev(&P->d_count, c->n_lanes) || !g.dev(&P->d_rows, kMaxStreamScans) || !g.pinned(&P->h_rows, kMaxStreamScans)) {
    delete P; return ALOAM_ERR_CUDA;
  }
  own(c, std::move(g));
  own(c, [P] { delete P; });
  c->place = P;
  return ALOAM_OK;
}

// room for n pairs in the pair scratch: a smaller one is replaced (the caller has drained the stream); a failure leaves it as it was
int pairs_reserve(Place* P, long long n) {
  if (P->pair_cap >= n) return ALOAM_OK;
  BufGroup g;
  double* dist; int* shift;
  if (!g.dev(&dist, (size_t)n) || !g.dev(&shift, (size_t)n)) return ALOAM_ERR_CUDA;
  P->pairs.swap(g);
  P->d_dist = dist; P->d_shift = shift; P->pair_cap = n;
  return ALOAM_OK;
}

PlaceSets db_sets(const Place* P) {
  PlaceSets S = {};
  S.rec = P->d_db; S.norm = P->d_db_norm; S.n = P->db_n; S.stream = false; S.dist = P->d_dist; S.shift = P->d_shift; S.stride = P->db_n;
  return S;
}

}  // namespace

int place_clear(aloam_ctx* c, int lane) {
  Place* P = c->place;
  if (!P || P->tables.empty()) return ALOAM_OK;
  const int l0 = lane < 0 ? 0 : lane, nl = lane < 0 ? c->n_lanes : 1;
  CUDA_CHECK_RET(cudaMemsetAsync(P->d_count + l0, 0, nl * sizeof(int), c->stream));
  for (int l = l0; l < l0 + nl; ++l) P->upper[l] = 0;
  return ALOAM_OK;
}

aloam_place_row* place_rows_device(aloam_ctx* c) { return c->place->d_rows; }
aloam_place_row* place_rows_host(aloam_ctx* c) { return c->place->h_rows; }

PlaceTable place_table(aloam_ctx* c, int lane) {
  const Place* P = c->place;
  return PlaceTable{P->d_rec + (size_t)lane * P->alloc * kRec, P->d_count + lane, P->cap, P->opt.exclude_recent};
}

int place_record_device(aloam_ctx* c, int nb, const MapperIn* in, const int* scan, const bool* start, aloam_place_row* const* rows, int* n_upper_out) {
  if (n_upper_out) *n_upper_out = 0;
  Place* P = c->place;
  if (nb < 1 || nb > ALOAM_MAX_BATCH || !P || P->tables.empty()) return ALOAM_ERR_STATE;
  Batch<PlaceGate> G = {};
  PlaceSets S = {};
  int n_upper = 0;   // the most candidates a record can query: its new keyframe's index is at most its lane's bound
  for (int l = 0; l < nb; ++l) {
    const int lane = in[l].lane;
    char* rec = P->d_rec + (size_t)lane * P->alloc * kRec;
    double* norm = P->d_norm + (size_t)lane * P->alloc * kSectors;
    G.a[l] = PlaceGate{in[l].corner, in[l].nc, in[l].surf, in[l].ns, in[l].out7, rec, norm, P->d_count + lane, rows[l], scan[l], lane, start[l] ? 1 : 0};
    if (start[l]) P->upper[lane] = 0;
    n_upper = std::max(n_upper, std::min(P->upper[lane], P->cap - 1) - P->opt.exclude_recent);
    P->upper[lane] = std::min(P->cap, P->upper[lane] + 1);
    S.s.a[l] = PlaceSet{nullptr, rec, norm, 0, rows[l]};
  }
  const double gap2 = P->opt.keyframe_gap * P->opt.keyframe_gap;
  LAUNCH(c, KID_PLACE_GATE, k_place_gate, nb, kDescThreads, 0, G, P->cap, P->opt.max_range, P->opt.z_offset, gap2);
  CUDA_CHECK_RET(cudaGetLastError());
  if (n_upper_out) *n_upper_out = n_upper;
  if (n_upper <= 0) return ALOAM_OK;   // no record has an older keyframe to query: the rows keep the gate's -1 fields
  S.exclude = P->opt.exclude_recent; S.stream = true;
  S.dist = P->d_dist; S.shift = P->d_shift; S.stride = P->alloc;
  LAUNCH(c, KID_PLACE_DIST, k_place_dist, dim3((n_upper + kDistPairs - 1) / kDistPairs, nb), kDistPairs * 64, place_dist_smem(), S);
  LAUNCH(c, KID_PLACE_BEST, k_place_best, nb, kBestThreads, 0, S, 1, nullptr);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

extern "C" {

int aloam_set_place(aloam_ctx* c, int on, const aloam_place_opts* opts) {
  if (!c || !opts || (on != 0 && on != 1)) return ALOAM_ERR_INVALID_ARG;
  const aloam_place_opts o = *opts;
  if (!std::isfinite(o.max_range) || !std::isfinite(o.z_offset) || !std::isfinite(o.keyframe_gap) || !(o.max_range > 0.f) ||
      !(o.keyframe_gap >= 0.0) || o.exclude_recent < 0 || o.max_keyframes < 1 || o.max_keyframes > kMaxKeyframes)
    return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c)) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (int rc = place_ensure(c)) return rc;
  Place* P = c->place;
  if (on && P->alloc < o.max_keyframes) {   // the tables of every lane, and the loop query's pairs
    const size_t L = c->n_lanes, K = o.max_keyframes;
    BufGroup tables;
    char* rec; double* norm;
    if (!tables.dev(&rec, L * K * kRec) || !tables.dev(&norm, L * K * kSectors)) return ALOAM_ERR_CUDA;
    // the loop query's pairs share the database query's scratch (nothing runs on it between calls)
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
    if (int rc = pairs_reserve(P, (long long)(L * K))) return rc;
    P->tables.swap(tables);   // no frame reads the old tables: every stream call drains before it returns
    P->d_rec = rec; P->d_norm = norm; P->alloc = o.max_keyframes;
  }
  P->opt = o;
  P->cap = std::min(o.max_keyframes, P->alloc);
  c->loop_on = false;   // the keyframe clouds belong to the tables this call clears (aloam_set_loops turns them on again)
  if (!P->tables.empty()) {
    CUDA_CHECK_RET(cudaMemsetAsync(P->d_count, 0, c->n_lanes * sizeof(int), c->stream));
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
    for (int& u : P->upper) u = 0;
  }
  c->place_on = on == 1;
  return ALOAM_OK;
}

int aloam_place_rows(aloam_ctx* c, aloam_place_row* out, int rows) {
  if (!c || !out) return ALOAM_ERR_INVALID_ARG;
  const MappedCall& M = c->last_mapped;
  if (const int rc = M.check(M.places, rows)) return rc;
  for (int r = 0; r < rows; ++r)
    out[r] = row_kind(M.table.rows[r]) == ALOAM_ROW_MAPPED ? c->place->h_rows[r] : aloam_place_row{-1, -1, -1, 0, -1.0};
  return ALOAM_OK;
}

int aloam_place_keyframes(aloam_ctx* c, int lane, void* out, long long capacity, long long* n_out) {
  if (!c || !n_out || lane < 0 || lane >= c->n_lanes || capacity < 0 || (capacity > 0 && !out)) return ALOAM_ERR_INVALID_ARG;
  const Place* P = c->place;
  if (!P || P->tables.empty()) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  int n = 0;
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (c->s_map) CUDA_CHECK_RET(cudaStreamSynchronize(c->s_map));
  CUDA_CHECK_RET(cudaMemcpy(&n, P->d_count + lane, sizeof(int), cudaMemcpyDeviceToHost));
  *n_out = n;
  if (capacity < n) return out || capacity ? ALOAM_ERR_CAPACITY : ALOAM_OK;
  if (n > 0) CUDA_CHECK_RET(cudaMemcpy(out, P->d_rec + (size_t)lane * P->alloc * kRec, (size_t)n * kRec, cudaMemcpyDefault));
  return ALOAM_OK;
}

int aloam_place_db_load(aloam_ctx* c, const void* records, int n_records) {
  if (!c || !records || n_records < 1 || n_records > kMaxDb) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (int rc = place_ensure(c)) return rc;
  Place* P = c->place;
  BufGroup db;
  char* rec; double* norm;
  if (!db.dev(&rec, (size_t)n_records * kRec) || !db.dev(&norm, (size_t)n_records * kSectors)) return ALOAM_ERR_CUDA;
  int err = 0;
  cudaError_t e = cudaMemcpyAsync(rec, records, (size_t)n_records * kRec, cudaMemcpyDefault, c->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(P->d_err, 0, sizeof(int), c->stream);
  if (e == cudaSuccess) { ++c->launches; k_place_load<<<n_records, 64, 0, c->stream>>>(rec, norm, bits_of(P->opt.max_range), bits_of(P->opt.z_offset), P->d_err); e = cudaGetLastError(); }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&err, P->d_err, sizeof(int), cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess || err) {
    cudaGetLastError();
    return e != cudaSuccess ? ALOAM_ERR_CUDA : ALOAM_ERR_INVALID_ARG;
  }
  P->db.swap(db);
  P->d_db = rec; P->d_db_norm = norm; P->db_n = n_records;
  return ALOAM_OK;
}

int aloam_place_db_clear(aloam_ctx* c) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  Place* P = c->place;
  if (!P || !P->d_db) return ALOAM_OK;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  P->db = BufGroup();
  P->d_db = nullptr; P->d_db_norm = nullptr; P->db_n = 0;
  return ALOAM_OK;
}

int aloam_place_describe(aloam_ctx* c, aloam_cloud_view less_sharp, aloam_cloud_view less_flat, float* desc) {
  if (!c || !desc) return ALOAM_ERR_INVALID_ARG;
  if (int rc = check_view(less_sharp)) return rc;
  if (int rc = check_view(less_flat)) return rc;
  if (less_sharp.n > c->max_points || less_flat.n > c->max_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (int rc = place_ensure(c)) return rc;
  Place* P = c->place;
  if (P->describe.empty()) {
    BufGroup g;
    Pt4* cloud[2]; float* desc;
    if (!g.dev(&cloud[0], c->max_points) || !g.dev(&cloud[1], c->max_points) || !g.dev(&desc, kBins)) return ALOAM_ERR_CUDA;
    P->describe.swap(g);
    P->d_cloud[0] = cloud[0]; P->d_cloud[1] = cloud[1]; P->d_desc = desc;
  }
  if (int rc = upload_cloud(c, less_sharp, P->d_cloud[0], c->max_points)) return rc;
  if (int rc = upload_cloud(c, less_flat, P->d_cloud[1], c->max_points)) return rc;
  LAUNCH(c, KID_PLACE_GATE, k_place_describe, 1, kDescThreads, 0, P->d_cloud[0], less_sharp.n, P->d_cloud[1], less_flat.n, P->opt.max_range,
         P->opt.z_offset, P->d_desc);
  CUDA_CHECK_RET(cudaGetLastError());
  CUDA_CHECK_RET(cudaMemcpyAsync(desc, P->d_desc, kBins * sizeof(float), cudaMemcpyDefault, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  return ALOAM_OK;
}

int aloam_place_query(aloam_ctx* c, const float* descs, int n_query, int k, aloam_place_match* out) {
  if (!c || !descs || !out || n_query < 1) return ALOAM_ERR_INVALID_ARG;
  Place* P = c->place;
  if (!P || !P->d_db) return ALOAM_ERR_STATE;
  if (k < 1 || k > std::min(ALOAM_PLACE_MAX_K, P->db_n)) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const int M = P->db_n;
  const int chunk = (int)std::max(1LL, std::min((long long)n_query, kMaxPairs / M));   // queries per launch pair
  const long long need_q = (long long)n_query * kBins, need_m = (long long)n_query * k;
  if (P->q_cap < need_q || P->match_cap < need_m) {   // either buffer grown to what this call needs, the other kept at its size
    BufGroup g;
    const long long q_cap = std::max(P->q_cap, need_q), match_cap = std::max(P->match_cap, need_m);
    float* q; aloam_place_match* match;
    if (!g.dev(&q, (size_t)q_cap) || !g.dev(&match, (size_t)match_cap)) return ALOAM_ERR_CUDA;
    P->query.swap(g);
    P->d_q = q; P->q_cap = q_cap; P->d_match = match; P->match_cap = match_cap;
  }
  if (P->pair_cap < (long long)chunk * M) {
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
    if (int rc = pairs_reserve(P, (long long)chunk * M)) return rc;
  }
  CUDA_CHECK_RET(cudaMemcpyAsync(P->d_q, descs, (size_t)n_query * kBins * sizeof(float), cudaMemcpyDefault, c->stream));
  for (int q0 = 0; q0 < n_query; q0 += chunk) {
    const int nq = std::min(chunk, n_query - q0);
    PlaceSets S = db_sets(P);
    S.q = P->d_q + (size_t)q0 * kBins;
    LAUNCH(c, KID_PLACE_DIST, k_place_dist, dim3((M + kDistPairs - 1) / kDistPairs, nq), kDistPairs * 64, place_dist_smem(), S);
    LAUNCH(c, KID_PLACE_BEST, k_place_best, nq, kBestThreads, 0, S, k, P->d_match + (size_t)q0 * k);
    CUDA_CHECK_RET(cudaGetLastError());
  }
  CUDA_CHECK_RET(cudaMemcpyAsync(out, P->d_match, (size_t)n_query * k * sizeof(aloam_place_match), cudaMemcpyDefault, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  return ALOAM_OK;
}

}  // extern "C"
