// Recovery of localising lanes inside the mapped stream calls (aloam_set_recovery, aloam_recovery_rows): when a localising row's
// prior-map inlier score (the tracking score, rows.cu) falls below trigger_frac of its scoring points, the same stream scores pose
// candidates around the row's map pose and, when the best one is clearly better, re-seats the lane's T_wmap_wodom.  The lane's next
// registered frame refines from there; its odometry goes on untouched.  Four launches per localising frame, whether or not a row
// triggers, all on the mapper stream right after the tracking score and decided on the device:
//   * k_recover_cand: per record the trigger test on its row (rec_triggered), then, for a triggered row only, candidate h =
//     (normalise(q_delta_h * q_P), t_P + t_delta_h) around the row's map pose P into the lane's slice -- an untriggered record's
//     CTAs leave at once;
//   * k_reloc_score / k_reloc_topk (reloc.cu), gated on rec_triggered: the candidates' coarse scores on the frame's filtered
//     stacks at the rows' scoring setting, and each set's best key, ranking by (score descending, h ascending).  The row's score
//     (k_inlier_score) and the candidates' count their points through the same walk (warp_inliers, grid.cuh), so a candidate at
//     the row's own pose ties with the row and the adoption's strict comparison never takes it;
//   * k_recover_adopt (cubemap.cu): the accept test and transformUpdate at the best candidate with the frame's odometry pose.
// Everything of a lane lives in the lane's slice of the buffers, so the scores of its latest triggered row stay readable.
#include "ctx.h"
#include "quat.cuh"

// the setting and the buffers, created by the first aloam_set_recovery that turns recovery on and replaced by larger ones as later
// calls need (one group); per lane l a slice of `cap` candidates, scores, ctas x kRelocTop CTA keys and kRelocTop best keys
struct aloam::Recovery {
  float trigger_frac = 0.f, accept_frac = 0.f;
  int n_delta = 0, cap = 0;
  int ctas = 0, ctas_cap = 0;                // CTAs of a record's k_reloc_score launch; the key slices are sized for ctas_cap
  BufGroup mem;
  double* d_delta = nullptr;                 // [cap][7] normalised deltas
  double* d_cand = nullptr;                  // [ALOAM_MAX_BATCH][cap][7]
  int* d_score = nullptr;                    // [ALOAM_MAX_BATCH][cap]
  unsigned long long* d_part = nullptr;      // [ALOAM_MAX_BATCH][ctas_cap * kRelocTop]
  unsigned long long* d_best = nullptr;      // [ALOAM_MAX_BATCH][kRelocTop]
  bool scored[ALOAM_MAX_BATCH] = {};         // the lane's slice holds the scores of a triggered row of the last mapped stream call
};

namespace {
constexpr int kMaxDelta = 65536;
constexpr int kCandThreads = 256;

// one record of k_recover_cand: the row, its map pose and the lane's candidate slice
struct RecoverCand {
  MapRowRec* row;
  const double* pose;
  double* cand;
};

// grid (candidate blocks, 1, records): the trigger test on the record's row -- n_score > 0 and (float)score < trigger_frac *
// (float)n_score -- written by thread 0 of CTA 0; a triggered record's candidates: h = (q_d * q_P normalised as
// map_pose_normalise (ctx.h) normalises, t_P + t_d) for the row's map pose P and delta d = delta[h]
__global__ void __launch_bounds__(kCandThreads) k_recover_cand(const __grid_constant__ Batch<RecoverCand> B, const double* __restrict__ delta, int n,
                                                             float trigger_frac) {
  const RecoverCand& a = B.a[blockIdx.z];
  const int score = a.row->score, n_score = a.row->n_score;
  const bool trig = n_score > 0 && (float)score < trigger_frac * (float)n_score;
  if (blockIdx.x == 0 && threadIdx.x == 0) a.row->rec_triggered = trig;
  if (!trig) return;   // CTA-uniform
  const int h = blockIdx.x * kCandThreads + threadIdx.x;
  if (h >= n) return;
  const double* d = delta + (size_t)h * 7;
  const double* P = a.pose;
  const Qd q = qmul(Qd{d[0], d[1], d[2], d[3]}, Qd{P[0], P[1], P[2], P[3]});
  const double qv[4] = {q.x, q.y, q.z, q.w};
  double n2 = 0;
  for (int k = 0; k < 4; ++k) n2 += qv[k] * qv[k];
  const double nrm = sqrt(n2);
  double* o = a.cand + (size_t)h * 7;
  for (int k = 0; k < 4; ++k) o[k] = qv[k] / nrm;
  for (int k = 0; k < 3; ++k) o[4 + k] = P[4 + k] + d[4 + k];
}

// room for n candidates and `ctas` CTA key lists per lane (a failure leaves the buffers as they were)
int recover_ensure(aloam_ctx* c, int n, int ctas) {
  if (!c->recover) {
    Recovery* R = new (std::nothrow) Recovery();
    if (!R) return ALOAM_ERR_CUDA;
    own(c, [R] { delete R; });
    c->recover = R;
  }
  Recovery* R = c->recover;
  if (n <= R->cap && ctas <= R->ctas_cap) return ALOAM_OK;
  const int cap = std::max(n, R->cap), ctas_cap = std::max(ctas, R->ctas_cap);
  BufGroup g;
  double *delta, *cand;
  int* score;
  unsigned long long *part, *best;
  const size_t L = ALOAM_MAX_BATCH;
  if (!g.dev(&delta, (size_t)cap * 7) || !g.dev(&cand, L * cap * 7) || !g.dev(&score, L * cap) || !g.dev(&part, L * ctas_cap * kRelocTop) ||
      !g.dev(&best, L * kRelocTop))
    return ALOAM_ERR_CUDA;
  R->mem.swap(g);
  R->d_delta = delta; R->d_cand = cand; R->d_score = score; R->d_part = part; R->d_best = best;
  R->cap = cap; R->ctas_cap = ctas_cap;
  return ALOAM_OK;
}

}  // namespace

// the recovery of the nb localising records of the frame just issued on the current stream (the mapper stream), after
// the tracking score has scored their rows rows[l]: four launches whatever the rows hold
int recover_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows) {
  const Recovery* R = c->recover;
  if (nb < 1 || nb > ALOAM_MAX_BATCH || !R || !c->prior) return ALOAM_ERR_STATE;
  Batch<RecoverCand> C = {};
  Batch<RelocRec> S = {};
  const double* cand[ALOAM_MAX_BATCH];
  const unsigned long long* best[ALOAM_MAX_BATCH];
  for (int l = 0; l < nb; ++l) {
    const int lane = in[l].lane;
    double* cs = R->d_cand + (size_t)lane * R->cap * 7;
    const FrameView F = frame_view(lane_frame(c, lane, true));
    C.a[l] = RecoverCand{rows[l], in[l].out7, cs};
    S.a[l] = RelocRec{cs, R->n_delta, {F.stack[0], F.stack[1]}, F.counts, R->d_score + (size_t)lane * R->cap,
                      R->d_part + (size_t)lane * R->ctas_cap * kRelocTop, R->d_best + (size_t)lane * kRelocTop, &rows[l]->rec_triggered};
    cand[l] = cs;
    best[l] = S.a[l].best;
  }
  LAUNCH(c, KID_RECOVER_CAND, k_recover_cand, dim3((R->n_delta + kCandThreads - 1) / kCandThreads, 1, nb), kCandThreads, 0, C, R->d_delta,
         R->n_delta, R->trigger_frac);
  reloc_score_device(c, nb, S, R->ctas, c->rows_max_score, c->rows_inlier_sq);
  reloc_topk_device(c, nb, S, R->ctas, 1);
  return recover_adopt_device(c, nb, in, rows, cand, best, R->accept_frac);
}

// which lanes' slices hold a triggered row of the last mapped stream call (its rows are in c->h_rows)
void recover_call_done(aloam_ctx* c) {
  Recovery* R = c->recover;
  if (!R) return;
  for (bool& s : R->scored) s = false;
  const MappedCall& M = c->last_mapped;
  if (!M.records || !M.recovered) return;
  for (int r = 0; r < M.n_scans * M.nb; ++r)
    if (row_kind(M.table.rows[r]) == ALOAM_ROW_LOCALISED && c->h_rows[r].rec_triggered) R->scored[r % M.nb] = true;
}

extern "C" {

int aloam_set_recovery(aloam_ctx* c, int on, const aloam_recovery_opts* opts, const double* deltas, int n_delta) {
  if (!c || (on != 0 && on != 1)) return ALOAM_ERR_INVALID_ARG;
  if (on == 0) {
    if (sharded_job(c)) return ALOAM_ERR_STATE;
    c->rec_on = false;
    return ALOAM_OK;
  }
  if (!opts || !deltas || n_delta < 1 || n_delta > kMaxDelta) return ALOAM_ERR_INVALID_ARG;
  const aloam_recovery_opts o = *opts;
  if (!(o.trigger_frac >= 0.f && o.trigger_frac <= 1.f) || !(o.accept_frac >= 0.f && o.accept_frac <= 1.f)) return ALOAM_ERR_INVALID_ARG;
  std::vector<double> d((size_t)n_delta * 7);
  for (size_t h = 0; h < (size_t)n_delta; ++h)
    if (!map_pose_normalise(deltas + 7 * h, deltas + 7 * h + 4, &d[7 * h])) return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c) || !c->rows_on || c->rows_max_score <= 0) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const int ctas = reloc_score_ctas(c, n_delta);
  const int rc = recover_ensure(c, n_delta, ctas); if (rc) return rc;
  Recovery* R = c->recover;
  CUDA_CHECK_RET(cudaMemcpy(R->d_delta, d.data(), d.size() * sizeof(double), cudaMemcpyHostToDevice));
  R->trigger_frac = o.trigger_frac;
  R->accept_frac = o.accept_frac;
  R->n_delta = n_delta;
  R->ctas = ctas;
  for (bool& s : R->scored) s = false;
  c->rec_on = true;
  return ALOAM_OK;
}

int aloam_recovery_rows(aloam_ctx* c, aloam_recovery_row* out, int rows) {
  if (!c || !out) return ALOAM_ERR_INVALID_ARG;
  const MappedCall& M = c->last_mapped;
  if (const int rc = M.check(M.records, rows)) return rc;
  for (int r = 0; r < rows; ++r) {
    aloam_recovery_row& o = out[r];
    std::memset(&o, 0, sizeof(o));
    o.best = o.best_score = -1;
    if (!M.recovered || row_kind(M.table.rows[r]) != ALOAM_ROW_LOCALISED) continue;
    const MapRowRec& h = c->h_rows[r];
    if (!h.rec_triggered) continue;
    o.triggered = 1;
    o.best = h.rec_best;
    o.best_score = h.rec_best_score;
    o.adopted = h.rec_adopted;
    for (int k = 0; k < 7; ++k) o.pose[k] = h.rec_pose[k];
  }
  return ALOAM_OK;
}

int aloam_debug_recovery_scores(aloam_ctx* c, int lane, int* scores, int n) {
  if (!c || !scores || lane < 0 || lane >= c->n_lanes) return ALOAM_ERR_INVALID_ARG;
  const Recovery* R = c->recover;
  if (!R || !R->scored[lane]) return ALOAM_ERR_STATE;
  if (n != R->n_delta) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaMemcpy(scores, R->d_score + (size_t)lane * R->cap, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  return ALOAM_OK;
}

}  // extern "C"
