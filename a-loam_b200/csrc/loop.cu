// Loop verification (include/aloam_b200.h: aloam_set_loops, aloam_loop_*, aloam_place_keyframe_cloud): the keyframe clouds of
// mapping lanes, and the registration of a keyframe against the submap of its loop candidate's neighbouring keyframes, in the
// mapped stream calls and on request.
//   * k_loop_keep: one CTA per record of a mapping frame, after k_place_gate.  It writes the row's "not verified" loop row; a
//     keyframe then copies the subsample of its lane's filtered stacks (the mapper's registration-set stacks, still in the sensor
//     frame after the frame: k_cube_ids writes the moved points elsewhere) into the lane's cloud pool at its keyframe index.
//   * k_loop_gather: grid (CTAs, 1, records).  A record runs when its place row has a candidate within max_distance (or always, for
//     aloam_loop_verify).  Every CTA builds the window's per-type offsets in shared memory and moves its share of the window's
//     stored points by their keyframe's pose into the submap buffers; it also copies the query keyframe's stored clouds into the
//     registration set's stacks.  CTA 0 writes the sizes, the thin test (a thin submap registers 0 queries, as k_mapper_prep
//     does, so the solve leaves the pose alone) and the initial pose.  An untriggered record writes zero sizes.
//   * then the mapper's own code: k_grid_setup + the K0 index build over the lanes' loop sets, map_register_device with the
//     verification's round count.
//   * the score: the relocaliser's inlier count of the query's stored points at the refined pose against the lane's registration
//     set's own grids, one launch of k_inlier_score (reloc.cu) with max_pts = cloud_points.  A stored cloud holds at most
//     cloud_points points per type, so every stored point is a scoring point, taken once.
//   * k_loop_finish: the constraint T_c^-1 * pose in Eigen's operation order, and the row (sizes, score, last round's summary head).
#include "ctx.h"
#include "quat.cuh"

namespace {
constexpr int kRec = ALOAM_PLACE_RECORD_BYTES;
constexpr int kMaxWindow = 64, kMaxSpan = 2 * kMaxWindow + 1;
constexpr int kMaxRounds = 16;
constexpr int kLoopThreads = 256;

// what a verification leaves on the device for the kernels after k_loop_gather (one per lane)
struct LoopState {
  int n_sub[2];      // submap sizes (corner, surf)
  int counts3[4];    // the registered stacks: n_corner, n_surf, total (0 for a thin submap)
  int n_q[2];        // the query keyframe's stored sizes (0 when the record is not verified): the score's points
  int active, query, cand, shift, thin, score;
  double pose[7];    // initial, then refined pose
};
}  // namespace

// one row of the loop-row table as the kernels leave it; aloam_loop_rows turns it into aloam_loop_row
struct LoopRowRec {
  int query, cand, verified, shift, n_sub[2], score, n_score, thin, pad;
  LmHead lm;         // the last round's summary head
  double pose[7], rel[7];
};

namespace {
// one lane's buffers: the cloud pool [cap][2][P] with its sizes [cap][2], a registration set sized for the submap bound and 2P
// queries (its stacks hold the query keyframe's clouds), the two submap buffers and the state
struct LoopLane {
  Pt4* pool;
  int* pool_n;
  MapReg reg;
  Pt4* sub[2];
  LoopState* st;
};
}  // namespace

struct aloam::Loop {
  aloam_loop_opts opt = {0.0, 0, 1, 1, 1.f};
  int cap = 0, bound = 0;                  // keyframes per lane in the pools; submap points per type, (2 window + 1) P
  std::vector<LoopLane> lanes;             // [n_lanes]
  BufGroup mem;                            // the per-lane buffers of the current setting
  double* d_rz = nullptr;                  // [60][2]: sin, cos of s * pi / 60, from the host's libm
  LoopRowRec* d_rows = nullptr;            // [kMaxStreamScans], and its pinned copy
  LoopRowRec* h_rows = nullptr;
  LoopRowRec* d_vrow = nullptr;            // the row of aloam_loop_verify, and its pinned copy
  LoopRowRec* h_vrow = nullptr;
};

namespace {

// ---- k_loop_keep: grid (records), kLoopThreads threads
struct LoopKeep {
  const aloam_place_row* prow;
  LoopRowRec* row;
  const Pt4* stack[2];
  const int* counts;
  Pt4* pool;
  int* pool_n;
};
__device__ __forceinline__ void row_unverified(LoopRowRec* r) {
  LoopRowRec z = {};
  z.query = z.cand = z.shift = -1;
  *r = z;
}
__global__ void __launch_bounds__(kLoopThreads) k_loop_keep(const __grid_constant__ Batch<LoopKeep> B, int P) {
  const LoopKeep& a = B.a[blockIdx.x];
  if (threadIdx.x == 0) row_unverified(a.row);
  const int kf = a.prow->keyframe;
  if (kf < 0) return;   // block-uniform
  for (int t = 0; t < 2; ++t) {
    const int n = a.counts[t], m = min(n, P);
    const Pt4* src = a.stack[t];
    Pt4* dst = a.pool + ((size_t)kf * 2 + t) * P;
    for (int i = threadIdx.x; i < m; i += blockDim.x) dst[i] = src[(long long)i * n / m];
    if (threadIdx.x == 0) a.pool_n[kf * 2 + t] = m;
  }
}

// ---- one record of a verification: the stream form reads (q, c, s) from its place row and runs when the row triggers; the
//      explicit form (prow null) always runs, from the pose init when has_init (already normalised) or else from shift s
struct LoopRec {
  const aloam_place_row* prow;
  const char* rec;        // the lane's keyframe records
  const Pt4* pool;
  const int* pool_n;
  Pt4* stack[2];
  Pt4* sub[2];
  LoopState* st;
  LoopRowRec* row;
  const LmSummary* summary;
  int q, c, s, has_init;
  double init[7];
};

// the pose normalisation of aloam_lane_localise (map_pose_normalise): |q|^2 summed in index order, q / sqrt
__device__ __forceinline__ void normalise_q(double* q) {
  double n2 = 0.0;
  for (int k = 0; k < 4; ++k) n2 += q[k] * q[k];
  const double n = sqrt(n2);
  for (int k = 0; k < 4; ++k) q[k] = q[k] / n;
}

// grid (CTAs, 1, records), kLoopThreads threads
__global__ void __launch_bounds__(kLoopThreads) k_loop_gather(const __grid_constant__ Batch<LoopRec> B, int P, int window, int exclude,
                                                              double max_distance, const double* __restrict__ rz) {
  const LoopRec& a = B.a[blockIdx.z];
  __shared__ int s_off[2][kMaxSpan + 1];
  __shared__ int s_hdr[5];   // active, q, c, lo, window size
  if (threadIdx.x == 0) {
    int q = a.q, cnd = a.c, act = 1;
    if (a.prow) { q = a.prow->keyframe; cnd = a.prow->loop; act = q >= 0 && cnd >= 0 && a.prow->distance <= max_distance; }
    const int lo = max(0, cnd - window), hi = min(cnd + window, q - 1 - exclude);
    s_hdr[0] = act; s_hdr[1] = q; s_hdr[2] = cnd; s_hdr[3] = lo; s_hdr[4] = act ? hi - lo + 1 : 0;
  }
  __syncthreads();
  LoopState* st = a.st;
  if (!s_hdr[0]) {   // block-uniform: nothing to register, nothing to score
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      st->active = 0; st->n_sub[0] = st->n_sub[1] = 0; st->n_q[0] = st->n_q[1] = 0; st->score = 0;
      st->counts3[0] = st->counts3[1] = st->counts3[2] = 0;
    }
    return;
  }
  const int q = s_hdr[1], cnd = s_hdr[2], lo = s_hdr[3], nw = s_hdr[4];
  for (int i = threadIdx.x; i < 2 * nw; i += blockDim.x) s_off[i & 1][(i >> 1) + 1] = a.pool_n[(lo + (i >> 1)) * 2 + (i & 1)];
  __syncthreads();
  if (threadIdx.x < 2) {
    const int t = threadIdx.x;
    s_off[t][0] = 0;
    for (int k = 0; k < nw; ++k) s_off[t][k + 1] += s_off[t][k];
  }
  __syncthreads();
  const int n0 = s_off[0][nw], n1 = s_off[1][nw];
  const int nq0 = a.pool_n[q * 2], nq1 = a.pool_n[q * 2 + 1];
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n0 + n1; j += stride) {
    const int t = j < n0 ? 0 : 1, i = j - (t ? n0 : 0);
    int k0 = 0, k1 = nw - 1;   // the last keyframe of the window whose points start at or before i
    while (k0 < k1) { const int mid = (k0 + k1 + 1) >> 1; if (s_off[t][mid] <= i) k0 = mid; else k1 = mid - 1; }
    const int kf = lo + k0;
    const double* x = reinterpret_cast<const double*>(a.rec + (size_t)kf * kRec);
    const Pt4 p = a.pool[((size_t)kf * 2 + t) * P + (i - s_off[t][k0])];
    a.sub[t][i] = point_associate_to_map(p, x[0], x[1], x[2], x[3], x[4], x[5], x[6]);
  }
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nq0 + nq1; j += stride) {
    const int t = j < nq0 ? 0 : 1, i = j - (t ? nq0 : 0);
    a.stack[t][i] = a.pool[((size_t)q * 2 + t) * P + i];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int thin = !(n0 > 10 && n1 > 50);   // laserMapping.cpp:554
    st->active = 1; st->query = q; st->cand = cnd; st->thin = thin; st->score = 0;
    st->n_sub[0] = n0; st->n_sub[1] = n1; st->n_q[0] = nq0; st->n_q[1] = nq1;
    st->counts3[0] = nq0; st->counts3[1] = nq1; st->counts3[2] = thin ? 0 : nq0 + nq1;
    if (a.prow ? false : a.has_init) {
      for (int k = 0; k < 7; ++k) st->pose[k] = a.init[k];
      st->shift = -1;
    } else {
      const int s = a.prow ? a.prow->shift : a.s;
      const double* xc = reinterpret_cast<const double*>(a.rec + (size_t)cnd * kRec);
      const double sz = rz[2 * s], cz = rz[2 * s + 1];
      const double x = xc[0], y = xc[1], z = xc[2], w = xc[3];
      double qq[4] = {x * cz + y * sz, y * cz - x * sz, z * cz + w * sz, w * cz - z * sz};   // q_c * Rz(s * 2 pi / 60)
      normalise_q(qq);
      for (int k = 0; k < 4; ++k) st->pose[k] = qq[k];
      for (int k = 4; k < 7; ++k) st->pose[k] = xc[k];
      st->shift = s;
    }
  }
}

// grid (records), 32 threads
__global__ void __launch_bounds__(32) k_loop_finish(const __grid_constant__ Batch<LoopRec> B, int last_round) {
  const LoopRec& a = B.a[blockIdx.x];
  const LoopState* st = a.st;
  if (threadIdx.x != 0 || !st->active) return;   // an untriggered row keeps what k_loop_keep wrote
  LoopRowRec r = {};
  r.query = st->query; r.cand = st->cand; r.verified = 1; r.shift = st->shift;
  r.n_sub[0] = st->n_sub[0]; r.n_sub[1] = st->n_sub[1];
  r.score = st->score; r.n_score = st->n_q[0] + st->n_q[1]; r.thin = st->thin;
  const LmSummary& s = a.summary[last_round & 3];
  r.lm = LmHead{s.termination, s.num_iterations, s.num_successful, s.num_jac_evals, s.n_edge, s.n_plane, s.initial_cost, s.final_cost};
  const double* xc = reinterpret_cast<const double*>(a.rec + (size_t)st->cand * kRec);
  for (int k = 0; k < 7; ++k) r.pose[k] = st->pose[k];
  const Qd cc{-xc[0], -xc[1], -xc[2], xc[3]};   // q_c.conjugate()
  const Qd qr = qmul(cc, Qd{r.pose[0], r.pose[1], r.pose[2], r.pose[3]});
  const double d[3] = {r.pose[4] - xc[4], r.pose[5] - xc[5], r.pose[6] - xc[6]};
  double t[3];
  qrot(cc, d, t);
  r.rel[0] = qr.x; r.rel[1] = qr.y; r.rel[2] = qr.z; r.rel[3] = qr.w;
  r.rel[4] = t[0]; r.rel[5] = t[1]; r.rel[6] = t[2];
  *a.row = r;
}

// the record of lane `lane` with its loop buffers (the place-row and verification fields are the caller's)
LoopRec lane_rec(aloam_ctx* c, int lane) {
  const Loop* Lp = c->loop;
  const LoopLane& L = Lp->lanes[lane];
  LoopRec r = {};
  r.rec = place_table(c, lane).rec;
  r.pool = L.pool; r.pool_n = L.pool_n;
  r.stack[0] = L.reg.stack[0]; r.stack[1] = L.reg.stack[1];
  r.sub[0] = L.sub[0]; r.sub[1] = L.sub[1];
  r.st = L.st; r.summary = L.reg.summary;
  return r;
}

// the launches of a verification of nb records (record l on lane lanes[l]) on c->stream: gather, index build, rounds, score, finish
int verify_device(aloam_ctx* c, int nb, const Batch<LoopRec>& B, const int* lanes) {
  const Loop* Lp = c->loop;
  const aloam_loop_opts& o = Lp->opt;
  const int P = o.cloud_points;
  const int G = std::max(1, std::min((2 * Lp->bound + 2 * P + kLoopThreads - 1) / kLoopThreads, std::max(1, c->sms * 4 / nb)));
  LAUNCH(c, KID_LOOP_VERIFY, k_loop_gather, dim3(G, 1, nb), kLoopThreads, 0, B, P, o.window, place_table(c, lanes[0]).exclude, o.max_distance,
         (const double*)Lp->d_rz);
  MapLaneIO io[ALOAM_MAX_BATCH];
  Batch<GridArgs> gs = {};
  Batch<ScoreRec> S = {};
  for (int l = 0; l < nb; ++l) {
    const LoopLane& L = Lp->lanes[lanes[l]];
    io[l] = MapLaneIO{L.reg, {L.sub[0], L.sub[1]}, L.st->counts3, L.st->pose};
    gs.a[l] = GridArgs{L.reg.corner.grid, L.sub[0], &L.st->n_sub[0], L.reg.surf.grid, L.sub[1], &L.st->n_sub[1]};
    S.a[l] = ScoreRec{{L.reg.stack[0], L.reg.stack[1]}, L.st->n_q, L.st->pose, {L.reg.corner.grid, L.reg.surf.grid}, &L.st->score};
  }
  launch_ex(c, KID_MAP_GRID, k_grid_setup, dim3(1, 1, nb), dim3(32), 0, 1, true, gs);
  map_index_build(c, nb, io, Lp->bound);
  if (const int rc = map_register_device(c, nb, io, 2 * P, o.outer_iters)) return rc;
  inlier_score_device(c, KID_LOOP_VERIFY, nb, S, 2LL * P, P, o.inlier_sq);
  LAUNCH(c, KID_LOOP_VERIFY, k_loop_finish, nb, 32, 0, B, o.outer_iters - 1);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

// the context's Loop with its row tables and heading table, created on first use and released by aloam_destroy
int loop_ensure(aloam_ctx* c) {
  if (c->loop) return ALOAM_OK;
  Loop* Lp = new (std::nothrow) Loop();
  if (!Lp) return ALOAM_ERR_CUDA;
  double rz[2 * ALOAM_PLACE_SECTORS];
  for (int s = 0; s < ALOAM_PLACE_SECTORS; ++s) {   // as place_hypotheses: a = s * 2 pi / 60, (sin, cos)(a / 2)
    const double a = (double)s * 2.0 * M_PI / ALOAM_PLACE_SECTORS;
    rz[2 * s] = std::sin(a / 2); rz[2 * s + 1] = std::cos(a / 2);
  }
  BufGroup g;
  const bool ok = g.dev(&Lp->d_rz, 2 * ALOAM_PLACE_SECTORS) && cudaMemcpy(Lp->d_rz, rz, sizeof(rz), cudaMemcpyHostToDevice) == cudaSuccess &&
                  g.dev(&Lp->d_rows, kMaxStreamScans) && g.pinned(&Lp->h_rows, kMaxStreamScans) && g.dev(&Lp->d_vrow, 1) && g.pinned(&Lp->h_vrow, 1);
  if (!ok) { cudaGetLastError(); delete Lp; return ALOAM_ERR_CUDA; }
  own(c, std::move(g));
  own(c, [Lp] { delete Lp; });
  c->loop = Lp;
  return ALOAM_OK;
}

// the per-lane buffers of a setting with pools of cap keyframes and P points per type (see the header's memory note); on
// failure nothing of the old setting has changed
int loop_alloc(aloam_ctx* c, int cap, int P, int bound) {
  Loop* Lp = c->loop;
  BufGroup g;
  std::vector<LoopLane> lanes(c->n_lanes);
  unsigned slots = 1024;
  while (slots < (unsigned)bound + ((unsigned)bound >> 2)) slots <<= 1;
  for (LoopLane& L : lanes) {
    L = LoopLane{};
    const bool ok = g.dev(&L.pool, (size_t)cap * 2 * P) && g.dev(&L.pool_n, (size_t)cap * 2) && g.dev(&L.sub[0], (size_t)bound) &&
                    g.dev(&L.sub[1], (size_t)bound) && g.dev(&L.st, 1) && map_reg_alloc(g, &L.reg, (size_t)2 * P, (size_t)bound, slots) == ALOAM_OK &&
                    cudaMemset(L.st, 0, sizeof(LoopState)) == cudaSuccess;
    if (!ok) { cudaGetLastError(); return ALOAM_ERR_CUDA; }
  }
  Lp->mem.swap(g);   // no frame reads the old buffers: every stream call drains before it returns
  Lp->lanes = std::move(lanes);
  Lp->cap = cap;
  Lp->bound = bound;
  return ALOAM_OK;
}

void row_out(const LoopRowRec& h, aloam_loop_row* o) {
  std::memset(o, 0, sizeof(*o));
  o->query = o->cand = o->shift = -1;
  if (!h.verified) return;
  o->query = h.query; o->cand = h.cand; o->verified = 1; o->shift = h.shift;
  o->n_sub[0] = h.n_sub[0]; o->n_sub[1] = h.n_sub[1];
  o->score = h.score; o->n_score = h.n_score;
  frame_stats_from(&h.lm, &o->stats, 1, h.thin ? ALOAM_FLAG_MAP_TOO_THIN : 0, 0.f);
  for (int k = 0; k < 7; ++k) { o->pose[k] = h.pose[k]; o->rel[k] = h.rel[k]; }
}

}  // namespace

void* loop_rows_device(aloam_ctx* c) { return c->loop->d_rows; }
void* loop_rows_host(aloam_ctx* c) { return c->loop->h_rows; }
size_t loop_row_bytes() { return sizeof(LoopRowRec); }

int loop_record_device(aloam_ctx* c, int nb, const MapperIn* in, const aloam_place_row* const* prow, size_t r0, int n_upper) {
  Loop* Lp = c->loop;
  if (nb < 1 || nb > ALOAM_MAX_BATCH || !Lp || Lp->lanes.empty()) return ALOAM_ERR_STATE;
  Batch<LoopKeep> K = {};
  Batch<LoopRec> B = {};
  int lanes[ALOAM_MAX_BATCH];
  for (int l = 0; l < nb; ++l) {
    const int lane = in[l].lane;
    const LoopLane& L = Lp->lanes[lane];
    const FrameView S = frame_view(lane_frame(c, lane, false));
    LoopRowRec* row = Lp->d_rows + r0 + lane;
    K.a[l] = LoopKeep{prow[l], row, {S.stack[0], S.stack[1]}, S.counts, L.pool, L.pool_n};
    B.a[l] = lane_rec(c, lane);
    B.a[l].prow = prow[l];
    B.a[l].row = row;
    lanes[l] = lane;
  }
  LAUNCH(c, KID_LOOP_KEEP, k_loop_keep, nb, kLoopThreads, 0, K, Lp->opt.cloud_points);
  CUDA_CHECK_RET(cudaGetLastError());
  if (n_upper <= 0) return ALOAM_OK;   // no record can have a candidate: every row keeps k_loop_keep's "not verified"
  return verify_device(c, nb, B, lanes);
}

extern "C" {

int aloam_set_loops(aloam_ctx* c, int on, const aloam_loop_opts* opts) {
  if (!c || !opts || (on != 0 && on != 1)) return ALOAM_ERR_INVALID_ARG;
  const aloam_loop_opts o = *opts;
  if (!(o.max_distance >= 0.0) || !std::isfinite(o.max_distance) || o.window < 0 || o.window > kMaxWindow || o.cloud_points < 1 ||
      o.cloud_points > c->cfg.max_points || o.outer_iters < 1 || o.outer_iters > kMaxRounds || !(o.inlier_sq > 0.f && o.inlier_sq <= 1.f))
    return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c)) return ALOAM_ERR_STATE;
  if (on && !c->place_on) return ALOAM_ERR_STATE;
  const long long bound = (2LL * o.window + 1) * o.cloud_points;
  if (on && bound > c->cfg.max_map_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (on) {
    if (int rc = loop_ensure(c)) return rc;
    const int cap = place_table(c, 0).cap;
    Loop* Lp = c->loop;
    if (Lp->lanes.empty() || Lp->cap != cap || Lp->opt.cloud_points != o.cloud_points || Lp->bound != (int)bound) {
      CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
      if (int rc = loop_alloc(c, cap, o.cloud_points, (int)bound)) return rc;
    }
    Lp->opt = o;
  }
  if (const int rc = place_clear(c, -1)) return rc;   // every lane's keyframe table, and with it its clouds
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  c->loop_on = on == 1;
  return ALOAM_OK;
}

int aloam_loop_rows(aloam_ctx* c, aloam_loop_row* out, int rows) {
  if (!c || !out) return ALOAM_ERR_INVALID_ARG;
  const MappedCall& M = c->last_mapped;
  if (const int rc = M.check(M.loops, rows)) return rc;
  const LoopRowRec none = {0, 0, 0};
  for (int r = 0; r < rows; ++r) row_out(row_kind(M.table.rows[r]) == ALOAM_ROW_MAPPED ? c->loop->h_rows[r] : none, &out[r]);
  return ALOAM_OK;
}

int aloam_loop_verify(aloam_ctx* c, int lane, int query, int cand, int shift, const double init[7], aloam_loop_row* out) {
  if (!c || !out || lane < 0 || lane >= c->n_lanes) return ALOAM_ERR_INVALID_ARG;
  double x0[7] = {};
  if (init && !map_pose_normalise(init, init + 4, x0)) return ALOAM_ERR_INVALID_ARG;
  if (!init && (shift < 0 || shift >= ALOAM_PLACE_SECTORS)) return ALOAM_ERR_INVALID_ARG;
  if (!c->loop_on) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (c->s_map) CUDA_CHECK_RET(cudaStreamSynchronize(c->s_map));
  const PlaceTable T = place_table(c, lane);
  int n = 0;
  CUDA_CHECK_RET(cudaMemcpy(&n, T.count, sizeof(int), cudaMemcpyDeviceToHost));
  if (query < 0 || query >= n || cand < 0 || cand > query - 1 - T.exclude) return ALOAM_ERR_INVALID_ARG;
  Loop* Lp = c->loop;
  Batch<LoopRec> B = {};
  B.a[0] = lane_rec(c, lane);
  B.a[0].prow = nullptr; B.a[0].row = Lp->d_vrow;
  B.a[0].q = query; B.a[0].c = cand; B.a[0].s = init ? -1 : shift; B.a[0].has_init = init ? 1 : 0;
  for (int k = 0; k < 7; ++k) B.a[0].init[k] = x0[k];
  const int lanes[1] = {lane};
  if (const int rc = verify_device(c, 1, B, lanes)) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(Lp->h_vrow, Lp->d_vrow, sizeof(LoopRowRec), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  row_out(*Lp->h_vrow, out);
  return ALOAM_OK;
}

int aloam_place_keyframe_cloud(aloam_ctx* c, int lane, int keyframe, float* out, long long capacity, long long n_out[2]) {
  if (!c || !n_out || lane < 0 || lane >= c->n_lanes || capacity < 0 || (capacity > 0 && !out)) return ALOAM_ERR_INVALID_ARG;
  if (!c->loop_on) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (c->s_map) CUDA_CHECK_RET(cudaStreamSynchronize(c->s_map));
  int n = 0;
  CUDA_CHECK_RET(cudaMemcpy(&n, place_table(c, lane).count, sizeof(int), cudaMemcpyDeviceToHost));
  if (keyframe < 0 || keyframe >= n) return ALOAM_ERR_INVALID_ARG;
  const LoopLane& L = c->loop->lanes[lane];
  const int P = c->loop->opt.cloud_points;
  int m[2] = {0, 0};
  CUDA_CHECK_RET(cudaMemcpy(m, L.pool_n + (size_t)keyframe * 2, sizeof(m), cudaMemcpyDeviceToHost));
  n_out[0] = m[0]; n_out[1] = m[1];
  if (capacity < (long long)m[0] + m[1]) return out || capacity ? ALOAM_ERR_CAPACITY : ALOAM_OK;
  for (int t = 0; t < 2; ++t)
    if (m[t] > 0)
      CUDA_CHECK_RET(cudaMemcpy(out + (t ? (size_t)m[0] * 4 : 0), L.pool + ((size_t)keyframe * 2 + t) * P, (size_t)m[t] * sizeof(Pt4), cudaMemcpyDefault));
  return ALOAM_OK;
}

}  // extern "C"
