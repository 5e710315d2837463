// Per-row records of the mapped stream calls (aloam_set_map_rows, aloam_map_rows): what each scan-to-map row of a call did, and
// for a localising row how well its scan still fits the prior map at the row's map pose.
//   * k_map_rows (cubemap.cu): one launch per frame, right after it on the mapper stream -- each record copies its frame's flags,
//     error word, window and stack sizes and the heads of its solve summaries into the row's slot of the device row table.
//   * k_track_score: the prior-map inlier score of aloam_prior_relocalise at the row's map pose, one launch per localising frame.
//     Parallel over the scoring points, not over records: grid (CTAs per record, 1, records), each warp takes 32 scoring points of
//     its record, lane j moves point j by the row's map pose (pointAssociateToMap in double), the warp walks the 32 moved points
//     through the cooperative 27-cell walk k_reloc_score uses (any_in_block27, grid.cuh) and adds its count to the row's score
//     with one atomic: an integer sum, so the score does not depend on the order the warps finish in.
//   * the host turns the rows into aloam_map_row after the call's final synchronise; skipped and idle rows cost no device work.
#include "ctx.h"
#include "grid.cuh"

namespace {
constexpr int kTrackWarps = 8;   // warps per CTA of k_track_score: 256 scoring points per CTA (at least 4 CTAs per SM: 46 registers, no spills)

// scores of the records' rows: row->score += the scoring points of the record's stacks (sizes counts[0], counts[1]; at most max_pts
// of each type, picked as k_reloc_score picks them) that have a prior-map point of their type at float d2 < inlier_sq once moved by
// the record's map pose.  Warps past the record's scoring points return at once.
__global__ void __launch_bounds__(kTrackWarps * 32, 4) k_track_score(const __grid_constant__ Batch<TrackArgs> B, int max_pts, float inlier_sq,
                                                                  const __grid_constant__ PriorGrid G) {
  const TrackArgs& a = B.a[blockIdx.z];
  const int n_c = a.counts[0], n_s = a.counts[1];
  const int m_c = min(n_c, max_pts), m_s = min(n_s, max_pts), m = m_c + m_s;
  const int p0 = (blockIdx.x * kTrackWarps + (threadIdx.x >> 5)) * 32;
  if (p0 >= m) return;   // warp-uniform
  const unsigned lane = lane_id();
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (p0 + (int)lane < m) {
    const float4 s = scoring_point(a.stack[0], a.stack[1], n_c, m_c, n_s, m_s, p0 + (int)lane);
    const double* x = a.pose;
    const Pt4 q = point_associate_to_map(Pt4{s.x, s.y, s.z, s.w}, x[0], x[1], x[2], x[3], x[4], x[5], x[6]);
    qx = q.x; qy = q.y; qz = q.z;
  }
  const unsigned mask_c = G.corner.dyn->mask, mask_s = G.surf.dyn->mask;
  const int np = min(32, m - p0);
  int cnt = 0;
  for (int j = 0; j < np; ++j) {
    const float px = __shfl_sync(0xffffffffu, qx, j), py = __shfl_sync(0xffffffffu, qy, j), pz = __shfl_sync(0xffffffffu, qz, j);
    const bool is_corner = p0 + j < m_c;
    const bool in = any_in_block27(is_corner ? G.corner : G.surf, is_corner ? mask_c : mask_s, px, py, pz,
                                   [&](float u, float v, float w) { return sqdist3(u, v, w, px, py, pz) < inlier_sq; });
    cnt += in ? 1 : 0;
  }
  if (lane == 0 && cnt) atomicAdd(&a.row->score, cnt);
}

}  // namespace

// k_track_score over the nb localising records of the frame just issued on the current stream, after k_map_rows has set their
// rows' counts to 0: record l scores rows[l] at its map pose in[l].out7 with its locator's filtered stacks.  The grid is sized
// from the host's bound on the scoring points, min(max_score, n_upper) per type.
int track_score_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, int n_upper_c, int n_upper_s) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH || !c->prior) return ALOAM_ERR_STATE;
  Batch<TrackArgs> B = {};
  for (int l = 0; l < nb; ++l) {
    const LocatorFrame F = locator_frame(c->lanes[in[l].lane].locator);
    B.a[l] = TrackArgs{{F.stack[0], F.stack[1]}, F.counts, in[l].out7, rows[l]};
  }
  const int max_pts = c->rows_max_score;
  const long long m_upper = (long long)std::min(max_pts, std::max(n_upper_c, 0)) + std::min(max_pts, std::max(n_upper_s, 0));
  const int ctas = (int)std::max(1LL, (m_upper + kTrackWarps * 32 - 1) / (kTrackWarps * 32));
  LAUNCH(c, KID_TRACK_SCORE, k_track_score, dim3(ctas, 1, nb), kTrackWarps * 32, 0, B, max_pts, c->rows_inlier_sq, prior_grid(c));
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
