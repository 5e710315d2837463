// Per-row records of the mapped stream calls (aloam_set_map_rows, aloam_map_rows): what each scan-to-map row of a call did, and
// for a localising row how well its scan still fits the prior map at the row's map pose.
//   * k_map_rows (cubemap.cu): one launch per frame, right after it on the mapper stream -- each record copies its frame's flags,
//     error word, window and stack sizes and the heads of its solve summaries into the row's slot of the device row table.
//   * the tracking score: the prior-map inlier score of aloam_prior_relocalise at the row's map pose, one launch of
//     k_inlier_score (reloc.cu) per localising frame, which counts the row's scoring points as k_reloc_score counts a hypothesis'.
//   * the host turns the rows into aloam_map_row after the call's final synchronise; skipped and idle rows cost no device work.
#include "ctx.h"

// the tracking score over the nb localising records of the frame just issued on the current stream, after k_map_rows has set
// their rows' counts to 0: record l scores rows[l] at its map pose in[l].out7 with its locator's filtered stacks against the prior
// map.  The grid is sized from the host's bound on the scoring points, min(max_score, n_upper) per type.
int track_score_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, int n_upper_c, int n_upper_s) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH || !c->prior) return ALOAM_ERR_STATE;
  const PriorGrid G = prior_grid(c);
  Batch<ScoreRec> B = {};
  for (int l = 0; l < nb; ++l) {
    const FrameView F = frame_view(lane_frame(c, in[l].lane, true));
    B.a[l] = ScoreRec{{F.stack[0], F.stack[1]}, F.counts, in[l].out7, {G.corner, G.surf}, &rows[l]->score};
  }
  const int max_pts = c->rows_max_score;
  const long long m_upper = (long long)std::min(max_pts, std::max(n_upper_c, 0)) + std::min(max_pts, std::max(n_upper_s, 0));
  inlier_score_device(c, KID_TRACK_SCORE, nb, B, m_upper, max_pts, c->rows_inlier_sq);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

extern "C" {

int aloam_set_map_rows(aloam_ctx* c, int on, float inlier_sq, int max_score_points) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  if ((on != 0 && on != 1) || max_score_points < 0 || (max_score_points > 0 && !(inlier_sq > 0.f && inlier_sq <= 1.f)))
    return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c)) return ALOAM_ERR_STATE;
  if (on && !c->d_rows) {   // first use: the row table and its pinned copy, kept until aloam_destroy
    CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
    MapRowRec *d = nullptr, *h = nullptr;
    if (dalloc(c, &d, (size_t)kMaxStreamScans) != cudaSuccess || halloc(c, &h, (size_t)kMaxStreamScans) != cudaSuccess) {
      cudaGetLastError();
      return ALOAM_ERR_CUDA;
    }
    c->d_rows = d; c->h_rows = h;
  }
  c->rows_on = on == 1;
  c->rows_inlier_sq = inlier_sq;
  c->rows_max_score = on ? max_score_points : 0;
  if (c->rows_max_score == 0) c->rec_on = false;   // recovery reads the rows' scores (aloam_set_recovery)
  return ALOAM_OK;
}

int aloam_map_rows(aloam_ctx* c, aloam_map_row* out, int rows) {
  if (!c || !out) return ALOAM_ERR_INVALID_ARG;
  const MappedCall& M = c->last_mapped;
  if (const int rc = M.check(M.records, rows)) return rc;
  for (int r = 0; r < rows; ++r) {
    aloam_map_row& o = out[r];
    std::memset(&o, 0, sizeof(o));
    o.kind = row_kind(M.table.rows[r]);
    if (o.kind == ALOAM_ROW_IDLE) continue;
    o.score = -1;
    if (o.kind == ALOAM_ROW_SKIPPED) continue;
    const MapRowRec& h = c->h_rows[r];
    o.err = h.err;
    o.n_valid = h.n_valid;
    for (int k = 0; k < 2; ++k) { o.n_sub[k] = h.n_sub[k]; o.n_stack[k] = h.n_stack[k]; }
    o.score = h.score;
    o.n_score = h.n_score;
    frame_stats_from(h.lm, &o.stats, c->cfg.outer_iters, h.flags, 0.f);
  }
  return ALOAM_OK;
}

}  // extern "C"
