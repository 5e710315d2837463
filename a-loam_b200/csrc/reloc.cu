// Relocalisation against the prior map (aloam_prior_relocalise): score many pose hypotheses of one scan against the whole prior
// map, keep the best K on the device, refine those with one batched localising frame.  Every inlier score of the library is
// taken here, by the two kernels below, and both count a warp's moved points with warp_inliers (grid.cuh).
//   * k_reloc_score: one warp per hypothesis, grid-stride over the hypotheses.  The scoring points (the frame's filtered stacks,
//     subsampled) are staged per CTA in shared memory with plain loads: they are a few KB read once per CTA, so a TMA bulk copy
//     would save nothing and needs a contiguous source, which the subsample is not.  Lane j moves point p0 + j by the warp's
//     hypothesis (pointAssociateToMap in double, once per point instead of 32 times), then warp_inliers walks the 32 moved points
//     in turn through the cooperative 27-cell walk of k_map_knn5 (lanes 0-26 probe one cell each, the candidates split over the
//     lanes 32 at a time), stopping after the first chunk in which some lane has a candidate inside inlier_sq.  The count stays
//     in a register; lane 0 writes it, and the warp keeps its 16 best keys (score << 32 | ~index) in lanes 0-15, merged per CTA
//     at the end.
//   * k_inlier_score: one pose per record (ScoreRec), parallel over the scoring points rather than the records -- the tracking
//     score of localising rows (rows.cu) and the score of a verified loop (loop.cu).  Grid (CTAs per record, 1, records), each
//     warp moves 32 scoring points of its record by the record's pose, counts them with warp_inliers and adds the count to the
//     record's score with one atomic: an integer sum, so the score does not depend on the order the warps finish in.
//   * k_reloc_topk: one CTA merges the per-CTA lists into the 16 best keys: ranking by (score descending, index ascending).
//   * both take one hypothesis set per record (RelocRec, blockIdx.z), with an optional device gate word: aloam_prior_relocalise is
//     the one-record, ungated case; the recovery of localising lanes (recover.cu) scores every localising record of a stream step
//     in one launch, gated on whether the record's row triggered.
//   * refinement: locate_step_device (cubemap.cu) over K records, each on a locator of the relocaliser's own, from T_wmap_wodom =
//     the hypothesis and the identity odometry pose: the first frame of a localising lane armed with that hypothesis.
#include <climits>
#include <vector>
#include "ctx.h"
#include "grid.cuh"

namespace {
constexpr int kRelocWarps = 8;                 // warps (hypotheses in flight) per CTA of k_reloc_score, 4 CTAs per SM (55 registers:
                                               // without the bound ptxas aims for 5 and spills the key list)
constexpr int kScoreWarps = 8;                 // warps per CTA of k_inlier_score: 256 scoring points per CTA (4 CTAs per SM:
                                               // 46 registers, no spills)
constexpr int kRelocStage = 2048;              // scoring points staged in shared memory at once (32 KB)
constexpr int kTop = kRelocTop;                // best keys kept per CTA and returned: the largest K
constexpr int kMaxHyp = 1 << 24;
}  // namespace

// The relocaliser's scratch, created on first use: the K locators (a localising lane's registration set each, context-owned,
// created as calls need them), the uploaded clouds and the per-call buffers.  The hypothesis buffers grow with the largest call
// (group `hyps`); the others are group `mem`.
struct aloam::Relocaliser {
  BufGroup mem, hyps;
  LaneFrame* loc[ALOAM_MAX_BATCH] = {};
  int n_loc = 0;
  Pt4* d_in[2] = {nullptr, nullptr};
  int* d_n = nullptr;                       // [2] the clouds' sizes
  double* d_hyp = nullptr;                  // [cap][7] normalised hypotheses
  int* d_score = nullptr;                   // [cap]
  long long cap = 0;
  int ctas = 0;                             // CTAs of a k_reloc_score launch over many hypotheses: one resident wave
  unsigned long long* d_part = nullptr;     // [ctas][kTop] per-CTA best keys
  unsigned long long* d_best = nullptr;     // [kTop]
  double* d_pose = nullptr;                 // [kTop][7] refined poses
  int* d_rscore = nullptr;                  // [kTop]
  struct Host { unsigned long long best[kTop]; int rscore[kTop]; double pose[kTop * 7]; int flags[kTop][2]; int n[2]; };
  Host* h = nullptr;                        // pinned
};

namespace {

// Scores of record blockIdx.z's set (RelocRec): score[h] of its n_hyp poses hyp[h] (7 doubles, q xyzw, t) = the scoring points of
// its stacks (sizes counts[0], counts[1]; at most max_pts of each type) that have a map point of their type at float d2 < inlier_sq.
// part (may be null): the CTA's kTop best keys (score << 32 | ~h), descending, 0 where there are fewer, at part[kTop * blockIdx.x].
// A gated set whose gate word is 0 leaves at once.
__global__ void __launch_bounds__(kRelocWarps * 32, 4) k_reloc_score(const __grid_constant__ Batch<RelocRec> B, int max_pts, float inlier_sq,
                                                                  const __grid_constant__ PriorGrid G) {
  const RelocRec& a = B.a[blockIdx.z];
  if (a.gate && !*a.gate) return;   // CTA-uniform
  const double* __restrict__ hyp = a.hyp;
  const Pt4* __restrict__ corner = a.stack[0];
  const Pt4* __restrict__ surf = a.stack[1];
  const int n_hyp = a.n_hyp;
  const int* counts = a.counts;
  __shared__ float4 s_pts[kRelocStage];
  __shared__ unsigned long long s_top[kRelocWarps * kTop], s_out[kTop];
  const int n_c = counts[0], n_s = counts[1];
  const int m_c = min(n_c, max_pts), m = scoring_points(n_c, n_s, max_pts), m_s = m - m_c;
  const unsigned lane = lane_id();
  const int warp = threadIdx.x >> 5;
  const unsigned mask_c = G.corner.dyn->mask, mask_s = G.surf.dyn->mask;
  const bool once = m <= kRelocStage;   // every scoring point fits: staged once for all of the CTA's hypotheses
  if (once) {
    for (int i = threadIdx.x; i < m; i += blockDim.x) s_pts[i] = scoring_point(corner, surf, n_c, m_c, n_s, m_s, i);
    __syncthreads();
  }
  unsigned long long top = 0;   // lanes 0 .. kTop-1: the warp's best keys so far, descending (0: none; every key is > 0)
  for (int h0 = blockIdx.x * kRelocWarps; h0 < n_hyp; h0 += gridDim.x * kRelocWarps) {   // CTA-uniform
    const int h = h0 + warp;
    const bool live = h < n_hyp;
    double x[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) x[k] = live ? hyp[(size_t)h * 7 + k] : 0.0;
    int cnt = 0;
    for (int c0 = 0; c0 < m; c0 += kRelocStage) {
      const int c1 = min(m, c0 + kRelocStage);
      if (!once) {
        __syncthreads();
        for (int i = c0 + threadIdx.x; i < c1; i += blockDim.x) s_pts[i - c0] = scoring_point(corner, surf, n_c, m_c, n_s, m_s, i);
        __syncthreads();
      }
      if (!live) continue;
      for (int p0 = c0; p0 < c1; p0 += 32) {
        float qx = 0.f, qy = 0.f, qz = 0.f;
        if (p0 + (int)lane < c1) {
          const float4 s = s_pts[p0 + lane - c0];
          const Pt4 q = point_associate_to_map(Pt4{s.x, s.y, s.z, s.w}, x[0], x[1], x[2], x[3], x[4], x[5], x[6]);
          qx = q.x; qy = q.y; qz = q.z;
        }
        cnt = warp_inliers(cnt, qx, qy, qz, p0, min(32, c1 - p0), m_c, G.corner, mask_c, G.surf, mask_s, inlier_sq);
      }
    }
    if (!live) continue;
    if (lane == 0) a.score[h] = cnt;
    // insert the key into the warp's descending list: the lanes that beat it stay, the others move one lane down
    const unsigned long long key = ((unsigned long long)(unsigned)cnt << 32) | (unsigned)~(unsigned)h;
    const int pos = __popc(__ballot_sync(0xffffffffu, top > key));
    const unsigned long long up = __shfl_up_sync(0xffffffffu, top, 1);
    if ((int)lane < kTop && (int)lane >= pos) top = (int)lane == pos ? key : up;
  }
  unsigned long long* best = a.part;
  if (!best) return;
  // the CTA's kTop best of its warps' lists: a key's rank is the number of keys above it (keys are unique, 0 is no key)
  if ((int)lane < kTop) s_top[warp * kTop + lane] = top;
  if (threadIdx.x < kTop) s_out[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x < kRelocWarps * kTop) {
    const unsigned long long k = s_top[threadIdx.x];
    int rank = 0;
    for (int i = 0; i < kRelocWarps * kTop; ++i) rank += s_top[i] > k;
    if (k && rank < kTop) s_out[rank] = k;
  }
  __syncthreads();
  if (threadIdx.x < kTop) best[(size_t)blockIdx.x * kTop + threadIdx.x] = s_out[threadIdx.x];
}

// scores of the records (ScoreRec): *score += the scoring points of the record's stacks (sizes counts[0], counts[1]; at most
// max_pts of each type) that have a map point of their type at float d2 < inlier_sq once moved by the record's pose.  Warp w of
// CTA b takes scoring points 32 (b kScoreWarps + w) .. + 31; warps past the record's scoring points return at once.
__global__ void __launch_bounds__(kScoreWarps * 32, 4) k_inlier_score(const __grid_constant__ Batch<ScoreRec> B, int max_pts, float inlier_sq) {
  const ScoreRec& a = B.a[blockIdx.z];
  const int n_c = a.counts[0], n_s = a.counts[1];
  const int m_c = min(n_c, max_pts), m = scoring_points(n_c, n_s, max_pts), m_s = m - m_c;
  const int p0 = (blockIdx.x * kScoreWarps + (threadIdx.x >> 5)) * 32;
  if (p0 >= m) return;   // warp-uniform
  const unsigned lane = lane_id();
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (p0 + (int)lane < m) {
    const float4 s = scoring_point(a.stack[0], a.stack[1], n_c, m_c, n_s, m_s, p0 + (int)lane);
    const double* x = a.pose;
    const Pt4 q = point_associate_to_map(Pt4{s.x, s.y, s.z, s.w}, x[0], x[1], x[2], x[3], x[4], x[5], x[6]);
    qx = q.x; qy = q.y; qz = q.z;
  }
  const unsigned mask_c = a.grid[0].dyn->mask, mask_s = a.grid[1].dyn->mask;
  const int cnt = warp_inliers(0, qx, qy, qz, p0, min(32, m - p0), m_c, a.grid[0], mask_c, a.grid[1], mask_s, inlier_sq);
  if (lane == 0 && cnt) atomicAdd(a.score, cnt);
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { const unsigned long long o = __shfl_xor_sync(0xffffffffu, v, d); v = o > v ? o : v; }
  return v;
}

// one CTA of 1024 per record (blockIdx.z): best[r] = the r-th largest of the n keys of its part (0 where there are fewer),
// r < rounds <= kTop -- `rounds` rounds of a block maximum over the keys below the previous round's.  A gated record whose gate
// word is 0 leaves at once.
__global__ void __launch_bounds__(1024) k_reloc_topk(const __grid_constant__ Batch<RelocRec> B, int n, int rounds) {
  const RelocRec& a = B.a[blockIdx.z];
  if (a.gate && !*a.gate) return;   // CTA-uniform
  const unsigned long long* __restrict__ part = a.part;
  unsigned long long* __restrict__ out = a.best;
  __shared__ unsigned long long s_w[32];
  unsigned long long prev = ~0ull;
  for (int r = 0; r < rounds; ++r) {
    unsigned long long m = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const unsigned long long k = part[i]; if (k < prev && k > m) m = k; }
    m = warp_max_u64(m);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = m;
    __syncthreads();
    m = warp_max_u64(threadIdx.x < 32 ? s_w[threadIdx.x & 31] : 0ull);
    m = __shfl_sync(0xffffffffu, m, 0);
    if (threadIdx.x == 0) s_w[0] = m;
    __syncthreads();
    prev = s_w[0];
    __syncthreads();
    if (threadIdx.x == 0) out[r] = prev;
  }
}

}  // namespace

void reloc_score_device(aloam_ctx* c, int nrec, const Batch<RelocRec>& B, int ctas, int max_pts, float inlier_sq) {
  LAUNCH(c, KID_RELOC, k_reloc_score, dim3(ctas, 1, nrec), kRelocWarps * 32, 0, B, max_pts, inlier_sq, prior_grid(c));
}

void reloc_topk_device(aloam_ctx* c, int nrec, const Batch<RelocRec>& B, int ctas, int rounds) {
  LAUNCH(c, KID_RELOC_TOPK, k_reloc_topk, dim3(1, 1, nrec), 1024, 0, B, ctas * kTop, rounds);
}

void inlier_score_device(aloam_ctx* c, int kid, int nb, const Batch<ScoreRec>& B, long long m_upper, int max_pts, float inlier_sq) {
  const int ctas = (int)std::max(1LL, (m_upper + kScoreWarps * 32 - 1) / (kScoreWarps * 32));
  LAUNCH(c, kid, k_inlier_score, dim3(ctas, 1, nb), kScoreWarps * 32, 0, B, max_pts, inlier_sq);
}

// one resident wave of k_reloc_score, at most one warp per hypothesis
int reloc_score_ctas(aloam_ctx* c, int n_hyp) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_reloc_score, kRelocWarps * 32, 0) != cudaSuccess) { cudaGetLastError(); per_sm = 1; }
  return std::max(1, std::min(c->sms * std::max(per_sm, 1), (n_hyp + kRelocWarps - 1) / kRelocWarps));
}

namespace {

// the relocaliser with at least `k` locators and room for n_hyp hypotheses (a failure leaves what exists as it was); it is
// published only complete, a failed first attempt freed at once
int reloc_ensure(aloam_ctx* c, int k, int n_hyp) {
  if (!c->reloc) {
    Relocaliser* R = new (std::nothrow) Relocaliser();
    if (!R) return ALOAM_ERR_CUDA;
    int per_sm = 0;
    bool ok = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_reloc_score, kRelocWarps * 32, 0) == cudaSuccess;
    R->ctas = c->sms * std::max(per_sm, 1);
    BufGroup& g = R->mem;
    ok = ok && g.dev(&R->d_in[0], (size_t)c->max_points) && g.dev(&R->d_in[1], (size_t)c->max_points);
    ok = ok && g.dev(&R->d_n, 2) && g.dev(&R->d_part, (size_t)R->ctas * kTop);
    ok = ok && g.dev(&R->d_best, kTop) && g.dev(&R->d_pose, kTop * 7);
    ok = ok && g.dev(&R->d_rscore, kTop) && g.pinned(&R->h, 1);
    if (!ok) { cudaGetLastError(); delete R; return ALOAM_ERR_CUDA; }
    own(c, [R] { delete R; });
    c->reloc = R;
  }
  Relocaliser* R = c->reloc;
  while (R->n_loc < k) {
    const int rc = locator_create(c, &R->loc[R->n_loc]); if (rc) return rc;
    ++R->n_loc;
  }
  if (n_hyp > R->cap) {
    BufGroup g;
    double* hyp;
    int* sc;
    if (!g.dev(&hyp, (size_t)n_hyp * 7) || !g.dev(&sc, (size_t)n_hyp)) return ALOAM_ERR_CUDA;
    R->hyps.swap(g);
    R->d_hyp = hyp; R->d_score = sc; R->cap = n_hyp;
  }
  return ALOAM_OK;
}

// the one-record, ungated set of aloam_prior_relocalise: n poses at d_pose scored on its stacks into d_score, best keys per CTA into
// part when it is set
RelocRec reloc_set(const Relocaliser* R, const FrameView& F, const double* d_pose, int n, int* d_score, unsigned long long* part) {
  return RelocRec{d_pose, n, {F.stack[0], F.stack[1]}, F.counts, d_score, part, R->d_best, nullptr};
}

}  // namespace

extern "C" int aloam_prior_relocalise(aloam_ctx* c, aloam_cloud_view less_sharp, aloam_cloud_view less_flat, const double* hyps, int n_hyp,
                                      const aloam_reloc_opts* opts, int* scores, aloam_reloc_result* out) {
  if (!c || !hyps || !opts || !out) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(less_sharp); if (rc) return rc;
  rc = check_view(less_flat); if (rc) return rc;
  const aloam_reloc_opts o = *opts;
  const int K = o.refine;
  if (n_hyp < 1 || n_hyp > kMaxHyp || !(o.inlier_sq > 0.f && o.inlier_sq <= 1.f) || o.max_score_points < 1 || K < 1 || K > ALOAM_MAX_BATCH || K > n_hyp)
    return ALOAM_ERR_INVALID_ARG;
  if (!c->prior || sharded_job(c)) return ALOAM_ERR_STATE;
  if (less_sharp.n > c->max_points || less_flat.n > c->max_points) return ALOAM_ERR_CAPACITY;
  std::vector<double> hyp((size_t)n_hyp * 7);
  for (size_t i = 0; i < (size_t)n_hyp; ++i)
    if (!map_pose_normalise(hyps + 7 * i, hyps + 7 * i + 4, &hyp[7 * i])) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  rc = reloc_ensure(c, K, n_hyp); if (rc) return rc;
  Relocaliser* R = c->reloc;
  Relocaliser::Host* H = R->h;
  // ---- upload; the scoring stacks are the stack filters of a localising frame, run on locator 0
  rc = upload_cloud(c, less_sharp, R->d_in[0], c->max_points); if (rc) return rc;
  rc = upload_cloud(c, less_flat, R->d_in[1], c->max_points); if (rc) return rc;
  H->n[0] = less_sharp.n; H->n[1] = less_flat.n;
  CUDA_CHECK_RET(cudaMemcpyAsync(R->d_n, H->n, 2 * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(R->d_hyp, hyp.data(), hyp.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  const int n_up_c = std::max(less_sharp.n, 1), n_up_s = std::max(less_flat.n, 1);
  MapperIn rec[ALOAM_MAX_BATCH];
  for (int r = 0; r < K; ++r) rec[r] = MapperIn{R->d_in[0], R->d_n, R->d_in[1], R->d_n + 1, c->d_ident, R->d_pose + 7 * r, 0, 1, 1};
  rc = locator_stacks_device(c, R->loc[0], rec[0], n_up_c, n_up_s); if (rc) return rc;
  const FrameView F = frame_view(R->loc[0]);
  // ---- coarse scores and the K best
  const int ctas = std::max(1, std::min(R->ctas, (n_hyp + kRelocWarps - 1) / kRelocWarps));
  Batch<RelocRec> B = {};
  B.a[0] = reloc_set(R, F, R->d_hyp, n_hyp, R->d_score, R->d_part);
  reloc_score_device(c, 1, B, ctas, o.max_score_points, o.inlier_sq);
  reloc_topk_device(c, 1, B, ctas, kTop);
  CUDA_CHECK_RET(cudaMemcpyAsync(H->best, R->d_best, sizeof(H->best), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  int win[ALOAM_MAX_BATCH], win_score[ALOAM_MAX_BATCH];
  LaneFrame* lp[ALOAM_MAX_BATCH];
  const double* init[ALOAM_MAX_BATCH];
  for (int r = 0; r < K; ++r) {
    win[r] = (int)~(unsigned)(H->best[r] & 0xffffffffull);
    win_score[r] = (int)(H->best[r] >> 32);
    lp[r] = R->loc[r];
    init[r] = &hyp[(size_t)win[r] * 7];
  }
  // ---- refinement: one localising frame per winner, all in one batch, then the refined poses scored by the same kernel
  rc = locate_step_device(c, K, rec, lp, init, n_up_c, n_up_s); if (rc) return rc;
  B.a[0] = reloc_set(R, F, R->d_pose, K, R->d_rscore, nullptr);
  reloc_score_device(c, 1, B, (K + kRelocWarps - 1) / kRelocWarps, o.max_score_points, o.inlier_sq);
  CUDA_CHECK_RET(cudaMemcpyAsync(H->pose, R->d_pose, sizeof(double) * 7 * K, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(H->rscore, R->d_rscore, sizeof(int) * K, cudaMemcpyDeviceToHost, c->stream));
  for (int r = 0; r < K; ++r) CUDA_CHECK_RET(cudaMemcpyAsync(H->flags[r], frame_view(R->loc[r]).flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  if (scores) CUDA_CHECK_RET(cudaMemcpy(scores, R->d_score, (size_t)n_hyp * sizeof(int), cudaMemcpyDeviceToHost));
  prof_collect(c);
  // out: (refined score descending, coarse rank ascending)
  int order[ALOAM_MAX_BATCH];
  for (int r = 0; r < K; ++r) order[r] = r;
  std::stable_sort(order, order + K, [&](int a, int b) { return H->rscore[a] > H->rscore[b]; });
  bool key_overflow = false;
  for (int i = 0; i < K; ++i) {
    const int r = order[i];
    aloam_reloc_result& res = out[i];
    res.hyp = win[r];
    res.score = win_score[r];
    res.refined_score = H->rscore[r];
    res.flags = H->flags[r][0] & ALOAM_FLAG_MAP_TOO_THIN;
    for (int k = 0; k < 7; ++k) res.pose[k] = H->pose[7 * r + k];
    key_overflow = key_overflow || (H->flags[r][1] & 1);
  }
  return key_overflow ? ALOAM_ERR_CAPACITY : ALOAM_OK;
}
