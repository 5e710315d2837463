// Host side of the C ABI (include/aloam_b200.h): context, device buffers, kernel sequencing.
// The reference's host code around the hot path is C++ (the ROS node bodies), so this layer is C++ too.
// No CPU fallback: every entry point runs the sm_90a kernels or returns an error.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <chrono>
#include <cstring>
#include <new>
#include <utility>
#include <vector>
#include "../../include/aloam_b200.h"
#include "kernels.h"

#include "ctx.h"

extern "C" {

int aloam_map_knn_impl(aloam_ctx* c, int which, aloam_cloud_view queries, int k, int* idx, float* sqdist);

void aloam_default_config(aloam_config* cfg, int n_scans) {
  if (!cfg) return;
  std::memset(cfg, 0, sizeof(*cfg));
  cfg->n_scans = n_scans;
  // launch/aloam_velodyne_VLP_16.launch:3-13, ..._HDL_32.launch:3-13, ..._HDL_64.launch:3-13
  if (n_scans == 64) { cfg->minimum_range = 5.0f; cfg->line_res = 0.4f; cfg->plane_res = 0.8f; }
  else { cfg->minimum_range = 0.3f; cfg->line_res = 0.2f; cfg->plane_res = 0.4f; }
  cfg->outer_iters = 2; cfg->inner_iters = 4; cfg->huber = 0.1;
  cfg->dist_sq_thresh = 25.0; cfg->nearby_scan = 2.5;
  cfg->device = 0; cfg->max_points = 400000; cfg->max_map_points = 0;
  cfg->max_batch = 1; cfg->distortion = 0; cfg->max_ring_points = ALOAM_MAX_RING_POINTS;
  cfg->mapping_skip_frame = 1;
}

const char* aloam_strerror(int code) {
  switch (code) {
    case ALOAM_OK: return "ok";
    case ALOAM_ERR_INVALID_ARG: return "invalid argument";
    case ALOAM_ERR_UNSUPPORTED_SCANS: return "n_scans must be 16, 32 or 64 for elevation rings, 1..64 for driver rings (1..128 through aloam_create_wide)";
    case ALOAM_ERR_EMPTY_CLOUD: return "no point survives the NaN / minimum-range filter";
    case ALOAM_ERR_CAPACITY: return "cloud larger than the context capacity";
    case ALOAM_ERR_CUDA: return "CUDA error";
    case ALOAM_ERR_NO_DEVICE: return "no CUDA device";
    case ALOAM_ERR_RING_TOO_LARGE: return "a ring holds more than cfg.max_ring_points returns";
    case ALOAM_ERR_NOT_RING_MAJOR: return "a cloud's int(intensity) is not a ring, or falls two below an earlier one";
    case ALOAM_ERR_STATE: return "call sequence error";
    case ALOAM_ERR_COMM: return "communicator error";
    case ALOAM_ERR_SNAPSHOT: return "snapshot malformed, of another format version, or taken under a configuration that changes results";
    default: return "unknown error";
  }
}

int aloam_destroy(aloam_ctx* c) {
  if (!c) return ALOAM_OK;
  cudaSetDevice(c->cfg.device);
  for (cudaStream_t s : c->streams) cudaStreamSynchronize(s);
  for (auto r = c->release.rbegin(); r != c->release.rend(); ++r) (*r)();
  delete c;
  return ALOAM_OK;
}

int aloam_mapper_reset(aloam_ctx* c);

int aloam_reset_odometry(aloam_ctx* c) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const double ident[7] = {0, 0, 0, 1, 0, 0, 0};
  for (Lane& L : c->lanes) {
    CUDA_CHECK_RET(cudaMemcpyAsync(L.d_pose, ident, sizeof(ident), cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(L.d_world, ident, sizeof(ident), cudaMemcpyHostToDevice, c->stream));
  }
  if (const int rc = place_clear(c, -1)) return rc;   // every lane's keyframe table
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (c->s_idx) CUDA_CHECK_RET(cudaStreamSynchronize(c->s_idx));   // an index build of the last synchronous call may still be running
  c->frame = 0; c->have_last = false;
  c->lanes_mode = false;
  for (Lane& L : c->lanes) L.sched = LaneSched();
  return ALOAM_OK;
}

// aloam_create (max_field_rings 64) and aloam_create_wide (ALOAM_MAX_RINGS): the same context, only the range of driver rings differs
static int create_ctx(const aloam_config* cfg_in, aloam_ctx** out, int max_field_rings) {
  if (!cfg_in || !out) return ALOAM_ERR_INVALID_ARG;
  *out = nullptr;
  aloam_config cfg = *cfg_in;
  if (cfg.max_batch == 0) cfg.max_batch = 1;                                  // zero-initialised tail of an older caller
  if (cfg.max_ring_points == 0) cfg.max_ring_points = ALOAM_MAX_RING_POINTS;
  if (cfg.mapping_skip_frame == 0) cfg.mapping_skip_frame = 1;
  if (cfg.mapping_skip_frame < 0) return ALOAM_ERR_INVALID_ARG;
  if (cfg.ring_source != ALOAM_RING_ELEVATION && cfg.ring_source != ALOAM_RING_FIELD) return ALOAM_ERR_INVALID_ARG;
  if (cfg.ring_source == ALOAM_RING_FIELD ? cfg.n_scans < 1 || cfg.n_scans > max_field_rings : cfg.n_scans != 16 && cfg.n_scans != 32 && cfg.n_scans != 64)
    return ALOAM_ERR_UNSUPPORTED_SCANS;
  if (cfg.max_points <= 0 || cfg.outer_iters < 1 || cfg.outer_iters > 4 || cfg.inner_iters < 0) return ALOAM_ERR_INVALID_ARG;
  // the association index packs a point's index with its ring into a non-negative int (index << log2 W | ring) below INT_MAX,
  // which the search keeps as its "no candidate" word, and aloam_odometry_set_last takes clouds of up to max_points: indices
  // below 2^24 - 1 at W = 128, below 2^25 - 1 at W = 64
  const int ring_w = ring_width(cfg.n_scans);
  if (cfg.max_points > (ring_w > 64 ? (1 << 24) - 1 : (1 << 25) - 1)) return ALOAM_ERR_INVALID_ARG;
  if (!(cfg.nearby_scan >= 1.0)) return ALOAM_ERR_INVALID_ARG;   // the association's break tables need a window of +-1 ring at least
  // HuberLoss(a) needs a > 0, and a VoxelGrid leaf <= 0 or NaN has no voxels
  if (!(cfg.huber > 0) || !(cfg.line_res > 0) || !(cfg.plane_res > 0)) return ALOAM_ERR_INVALID_ARG;
  if (cfg.max_batch < 1 || cfg.max_batch > ALOAM_MAX_BATCH) return ALOAM_ERR_INVALID_ARG;
  if (cfg.max_ring_points < 64 || cfg.max_ring_points > ALOAM_MAX_RING_POINTS || cfg.max_ring_points % 32) return ALOAM_ERR_INVALID_ARG;
  if (cfg.max_map_points > (1 << 30)) return ALOAM_ERR_INVALID_ARG;   // the map's hash-grid slot count is a 32-bit power of two
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return ALOAM_ERR_NO_DEVICE;
  if (cfg.device < 0 || cfg.device >= ndev) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(cfg.device));
  aloam_ctx* c = new (std::nothrow) aloam_ctx();
  if (!c) return ALOAM_ERR_INVALID_ARG;
  c->cfg = cfg;
  c->max_points = cfg.max_points;
  c->max_ring = cfg.max_ring_points;
  c->ring_w = ring_w;
  c->n_lanes = cfg.max_batch;
  c->nblocks_max = (c->max_points + 1023) / 1024;
  const size_t mp = (size_t)c->max_points;
  const size_t mr = (size_t)c->max_ring;
  const size_t rw = (size_t)ring_w;   // the per-ring tables below hold rw rings: a 64-wide context allocates what it always did
#define TRY(e) do { if ((e) != cudaSuccess) { fprintf(stderr, "[aloam_b200] %s failed: %s\n", #e, cudaGetErrorString(cudaGetLastError())); aloam_destroy(c); return ALOAM_ERR_CUDA; } } while (0)
  TRY(cudaDeviceGetAttribute(&c->sms, cudaDevAttrMultiProcessorCount, cfg.device));
  TRY(screate(c, &c->stream));
  TRY(ecreate(c, &c->ev0, cudaEventDefault)); TRY(ecreate(c, &c->ev1, cudaEventDefault));
  for (cudaEvent_t& e : c->prof_ev) TRY(ecreate(c, &e, cudaEventDefault));
  for (cudaStream_t* s : {&c->s_ext, &c->s_h2d, &c->s_exa, &c->s_idx, &c->s_map}) TRY(screate(c, s));
  const std::pair<cudaEvent_t*, int> scan_events[] = {{c->ev_idx, kFeatSlots}, {c->ev_a, 2}, {c->ev_b, 2}, {c->ev_cmp, 2}, {c->ev_feat, kFeatSlots},
                                                      {c->ev_odo, kFeatSlots}, {c->ev_mapdone, kFeatSlots}, {c->ev_h2d, 2}, {c->ev_rawfree, 2},
                                                      {&c->ev_mapend, 1}};
  for (const auto& a : scan_events)
    for (int i = 0; i < a.second; ++i) TRY(ecreate(c, &a.first[i], cudaEventDisableTiming));
  TRY(halloc(c, &c->h_poses, (size_t)kMaxStreamScans * 14)); TRY(dalloc(c, &c->d_poses, (size_t)kMaxStreamScans * 7)); TRY(dalloc(c, &c->d_map_poses, (size_t)kMaxStreamScans * 7));
  TRY(halloc(c, &c->h_scan_nfull, (size_t)kMaxStreamScans)); TRY(dalloc(c, &c->d_scan_nfull, (size_t)kMaxStreamScans));
  TRY(dalloc(c, &c->d_curv, mp)); TRY(dalloc(c, &c->d_label, mp));
  c->lanes.resize(c->n_lanes);
  ScanScalars init[3];
  for (ScanScalars& s : init) { s.first_valid = INT32_MAX; s.last_valid = -1; s.half_idx = INT32_MAX; s.n_full = 0; s.start_ori = 0; s.end_ori = 0; s.error = 0; s.pad = 0; }
  for (Lane& L : c->lanes) {
    for (int b = 0; b < 2; ++b) {
      TRY(dalloc(c, &L.d_raw[b], mp * 8)); TRY(dalloc(c, &L.d_full[b], mp)); TRY(dalloc(c, &L.d_ring_start[b], rw + 8));
      TRY(dalloc(c, &L.st_sharp[b], rw * kMaxSharpPerRing)); TRY(dalloc(c, &L.st_less_sharp[b], rw * kMaxLessSharpPerRing));
      TRY(dalloc(c, &L.st_flat[b], rw * kMaxFlatPerRing)); TRY(dalloc(c, &L.st_less_flat[b], rw * mr));
      TRY(dalloc(c, &L.st_counts[b], rw * 4));
    }
    TRY(dalloc(c, &L.d_ring, mp));
    TRY(dalloc(c, &L.d_hist, (size_t)c->nblocks_max * rw)); TRY(dalloc(c, &L.d_offsets, (size_t)c->nblocks_max * rw));
    TRY(dalloc(c, &L.d_scan_start, rw)); TRY(dalloc(c, &L.d_scan_end, rw));
    TRY(dalloc(c, &L.d_sc, 3));
    TRY(cudaMemcpy(L.d_sc, init, sizeof(init), cudaMemcpyHostToDevice));
    for (FeatBuf& f : L.feat) {
      TRY(dalloc(c, &f.sharp, kMaxQueries)); TRY(dalloc(c, &f.flat, kMaxQueries));
      TRY(dalloc(c, &f.less_sharp, mp)); TRY(dalloc(c, &f.less_flat, mp));
      TRY(dalloc(c, &f.counts, 4));
      for (RabIndex* g : {&f.g_ls, &f.g_lf}) {
        TRY(dalloc(c, &g->cnt, (size_t)ALOAM_NB * rw)); TRY(dalloc(c, &g->start, (size_t)ALOAM_NB * rw + 8));
        TRY(dalloc(c, &g->cell_of, mp)); TRY(dalloc(c, &g->rank_of, mp)); TRY(dalloc(c, &g->gpts, mp));
        TRY(cudaMemset(g->cnt, 0, (size_t)ALOAM_NB * rw * 4)); TRY(cudaMemset(g->start, 0, ((size_t)ALOAM_NB * rw + 8) * 4));
        TRY(dalloc(c, &g->first_of, rab_break_ints(ring_w)));
        g->last_of = g->first_of + rw; g->fwd_end = g->last_of + rw; g->bwd_begin = g->fwd_end + rw + 1;
        TRY(cudaMemset(g->first_of, 0x7f, rw * 4)); TRY(cudaMemset(g->last_of, 0xff, rw * 4));   // 0x7f7f7f7f (> any index), -1
        TRY(cudaMemset(g->fwd_end, 0, (2 * rw + 2) * 4));
      }
      TRY(cudaMemset(f.counts, 0, 16));
    }
    TRY(dalloc(c, &L.d_blocks, (size_t)2 * kMaxQueries)); TRY(dalloc(c, &L.d_corr, (size_t)2 * kMaxQueries * 4));
    TRY(dalloc(c, &L.d_pose, 8)); TRY(dalloc(c, &L.d_world, 8)); TRY(dalloc(c, &L.d_summary, 4));
  }
  TRY(dalloc(c, &c->d_out28, 32)); TRY(dalloc(c, &c->d_api_pose, 8));
  TRY(dalloc(c, &c->d_ident, 7)); TRY(dalloc(c, &c->d_sc_init, 1));
  { const double ident[7] = {0, 0, 0, 1, 0, 0, 0};
    TRY(cudaMemcpy(c->d_ident, ident, sizeof(ident), cudaMemcpyHostToDevice));
    TRY(cudaMemcpy(c->d_sc_init, init, sizeof(ScanScalars), cudaMemcpyHostToDevice)); }
  TRY(dalloc(c, &c->d_packed, (size_t)2 * kMaxQueries * 11));
  TRY(dalloc(c, &c->d_err, 4));
  TRY(dalloc(c, &c->d_query, mp)); TRY(dalloc(c, &c->d_knn_idx, mp)); TRY(dalloc(c, &c->d_knn_d, mp));
  for (int k = 0; k < 5; ++k) TRY(halloc(c, &c->h_out[k], k == 0 || k == 4 ? mp : (size_t)kMaxQueries));
  TRY(halloc(c, &c->pin, 1));
  TRY(halloc(c, &c->h_summary, (size_t)4 * c->n_lanes)); TRY(halloc(c, &c->h_sc, (size_t)3 * c->n_lanes));
  TRY(cudaMemset(c->d_err, 0, 16));
  // function attributes are process-wide: always opt in to the largest ring capacity, whatever this context uses
  TRY(cudaFuncSetAttribute(k_ring_features, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring_features_smem_bytes(ALOAM_MAX_RING, true)));
  TRY(cudaFuncSetAttribute(k_ring_features_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring_features_smem_bytes(ALOAM_MAX_RING, false)));
  TRY(cudaFuncSetAttribute(k_lm_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lm_dynamic_smem_bytes()));
  TRY(cudaFuncSetAttribute(k_lm_solve_x, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lm_dynamic_smem_bytes()));
  TRY(cudaFuncSetAttribute(k_lm_eval_shard, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lm_dynamic_smem_bytes()));
#undef TRY
  int rc = aloam_reset_odometry(c);
  if (rc != ALOAM_OK) { aloam_destroy(c); return rc; }
  *out = c;
  return ALOAM_OK;
}

int aloam_create(const aloam_config* cfg, aloam_ctx** out) { return create_ctx(cfg, out, 64); }
int aloam_create_wide(const aloam_config* cfg, aloam_ctx** out) { return create_ctx(cfg, out, ALOAM_MAX_RINGS); }

}  // extern "C"

// ------------------------------------------------------------------------------------------------ kernel sequencing
namespace {

// Feature extraction is issued in two halves so that the pipelined stream call can run them on different streams:
//   A  ring binning   (k_classify, k_ring_scan, k_scatter)  raw scan -> ring-major cloud `full[buf]`, ring_start[buf]
//   B  per-ring work  (k_ring_features, k_compact)          full[buf] -> the four feature clouds of feat[slot]
// Every launch covers nb records; record l is the trajectory of lane pl[l] (the single-trajectory paths pass kLane0).
// Per-record arrays (d_raw, n) are indexed by record, per-lane ones by lane.  `sc_slot` (returned by A, consumed by B) is the
// ScanScalars parity slot of this scan; nfull_out (device, one int per lane, may be null) receives the ring-major cloud sizes.
constexpr int kLane0[1] = {0};
int run_features_a(aloam_ctx* c, int nb, const int* pl, const float* const* d_raw, const int* n, int stride, int buf, int* sc_slot, int* nfull_out) {
  int nmax = 0;
  for (int l = 0; l < nb; ++l) nmax = std::max(nmax, n[l]);
  const int blocks = (nmax + 1023) / 1024;
  const float thres = c->cfg.minimum_range;
  Batch<ClassifyArgs> ca = {}; Batch<RingScanArgs> ra = {}; Batch<ScatterArgs> sa = {};
  for (int l = 0; l < nb; ++l) {
    Lane& L = c->lanes[pl[l]];
    ScanScalars* sc = L.d_sc + c->parity;
    ScanScalars* sc_next = L.d_sc + (c->parity + 1) % 3;
    ca.a[l] = ClassifyArgs{d_raw[l], n[l], stride, L.d_ring, L.d_hist, sc};
    ra.a[l] = RingScanArgs{d_raw[l], stride, (n[l] + 1023) / 1024, L.d_hist, L.d_offsets, L.d_ring_start[buf], L.d_scan_start, L.d_scan_end, sc, sc_next,
                           nfull_out ? nfull_out + pl[l] : nullptr};
    sa.a[l] = ScatterArgs{d_raw[l], n[l], stride, L.d_ring, L.d_offsets, sc, L.d_full[buf]};
  }
  // one instance per (ring source, ring width); elevation rings stop at 64
  const auto classify = c->ring_w == 128 ? k_classify<ALOAM_RING_FIELD, 128>
                      : c->cfg.ring_source == ALOAM_RING_FIELD ? k_classify<ALOAM_RING_FIELD, 64> : k_classify<ALOAM_RING_ELEVATION, 64>;
  LAUNCH(c, KID_CLASSIFY, classify, dim3(blocks, nb), 256, 0, ca, c->cfg.n_scans, thres * thres);
  launch_ex(c, KID_RING_SCAN, c->ring_w == 128 ? k_ring_scan<128> : k_ring_scan<64>, dim3(nb), dim3(1024), 0, 1, true, ra, c->cfg.n_scans);
  launch_ex(c, KID_SCATTER, c->ring_w == 128 ? k_scatter<128> : k_scatter<64>, dim3(blocks, nb), dim3(256), 0, 1, true, sa);
  *sc_slot = c->parity;
  c->parity = (c->parity + 1) % 3;
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}
// B1: per-ring kernel -> staging set `buf` ; B2: ring-ordered concatenation of the staging set into feat[slot]
int run_features_b1(aloam_ctx* c, int nb, const int* pl, int buf, int sc_slot) {
  Batch<RingFeatArgs> fa = {};
  for (int l = 0; l < nb; ++l) {
    const int lane = pl[l];
    Lane& L = c->lanes[lane];
    fa.a[l] = RingFeatArgs{L.d_full[buf], L.d_ring_start[buf], L.st_sharp[buf], L.st_less_sharp[buf], L.st_flat[buf], L.st_less_flat[buf], L.st_counts[buf],
                           lane == 0 ? c->d_curv : nullptr, lane == 0 ? c->d_label : nullptr, L.d_sc + sc_slot};
  }
  // one trajectory: a cluster of two CTAs per ring (picks | voxel sort, see features.cu) ; a batch: one CTA per ring and trajectory
  if (nb == 1) launch_ex(c, KID_RING_FEATURES, k_ring_features, dim3(2 * c->cfg.n_scans, 1), dim3(512), ring_features_smem_bytes(c->max_ring, true), 2, false, fa, c->cfg.n_scans, 0.2f, c->max_ring);
  else LAUNCH(c, KID_RING_FEATURES, k_ring_features_batch, dim3(c->cfg.n_scans, nb), 256, ring_features_smem_bytes(c->max_ring, false), fa, c->cfg.n_scans, 0.2f, c->max_ring);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}
int run_features_b2(aloam_ctx* c, int nb, const int* pl, int buf, int slot, bool pdl) {
  Batch<CompactArgs> ka = {};
  for (int l = 0; l < nb; ++l) {
    Lane& L = c->lanes[pl[l]];
    FeatBuf& out = L.feat[slot];
    ka.a[l] = CompactArgs{L.st_sharp[buf], L.st_less_sharp[buf], L.st_flat[buf], L.st_less_flat[buf], L.st_counts[buf], out.sharp, out.less_sharp, out.flat,
                          out.less_flat, out.counts};
  }
  launch_ex(c, KID_COMPACT, k_compact, dim3(c->cfg.n_scans, nb), dim3(128), 0, 1, pdl, ka, c->cfg.n_scans, c->max_ring);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}
int run_features(aloam_ctx* c, const float* d_raw, int n, int stride, int slot) {
  int sc = 0;
  int rc = run_features_a(c, 1, kLane0, &d_raw, &n, stride, 0, &sc, nullptr);
  if (rc) return rc;
  rc = run_features_b1(c, 1, kLane0, 0, sc);
  if (rc) return rc;
  return run_features_b2(c, 1, kLane0, 0, slot, true);
}

// index over the two "last" clouds of feat[slot]: count -> scan -> fill (n_ls / n_lf = host upper bounds on the cloud sizes)
void run_grid_build(aloam_ctx* c, int nb, const int* pl, int slot, int n_ls, int n_lf) {
  const int pb = (std::max(std::max(n_ls, n_lf), 1) + 255) / 256;
  Batch<RabArgs> ga = {};
  for (int l = 0; l < nb; ++l) {
    FeatBuf& f = c->lanes[pl[l]].feat[slot];
    ga.a[l] = RabArgs{f.g_ls, f.less_sharp, f.counts + 1, f.g_lf, f.less_flat, f.counts + 3};
  }
  const bool wide = c->ring_w == 128;
  LAUNCH(c, KID_GRID_BUILD, (wide ? k_rab_count<128> : k_rab_count<64>), dim3(pb, 2, nb), 256, 0, ga);
  launch_ex(c, KID_GRID_BUILD, wide ? k_rab_scan<128> : k_rab_scan<64>, dim3(2, nb), dim3(1024), 0, 1, true, ga);
  launch_ex(c, KID_GRID_BUILD, wide ? k_rab_fill<128> : k_rab_fill<64>, dim3(pb, 2, nb), dim3(256), 0, 1, true, ga);
}

// outer_iters x (association + LM) ; feat[cur] supplies sharp/flat, feat[last] the targets ; pose in lane.d_pose
// pose_slots (device, lane-major 7 doubles each, may be null): the integrated world pose is also written there by the last solve
void run_register(aloam_ctx* c, int nb, const int* pl, int cur, int last, int sharp_slots, int flat_slots, bool integrate, bool want_corr,
                  double* pose_slots, double* pose_override /* may be null; record 0: solve for this pose instead of its lane's warm start */) {
  OdomParams op{c->cfg.dist_sq_thresh, c->cfg.nearby_scan, c->cfg.distortion};
  const LmParams lp = lm_params(c->cfg);
  const int slots = sharp_slots + flat_slots;
  for (int it = 0; it < c->cfg.outer_iters; ++it) {
    const bool last_it = it == c->cfg.outer_iters - 1;
    Batch<AssocArgs> aa = {}; Batch<LmArgs> la = {};
    for (int l = 0; l < nb; ++l) {
      const int lane = pl[l];
      Lane& L = c->lanes[lane];
      const FeatBuf& fc = L.feat[cur];
      const FeatBuf& fl = L.feat[last];
      double* pose = (l == 0 && pose_override) ? pose_override : L.d_pose;
      aa.a[l] = AssocArgs{fc.sharp, fc.flat, fc.counts, last_corner(fl), last_surf(fl), pose, L.d_blocks, want_corr ? L.d_corr : nullptr};
      la.a[l] = LmArgs{L.d_blocks, nullptr, slots, pose, L.d_summary + (it & 3), (integrate && last_it && pose_slots) ? pose_slots + (size_t)lane * 7 : nullptr, L.d_world};
    }
    // within one call the chain association -> LM -> association -> LM is launched with programmatic dependencies
    if (slots > 0) launch_ex(c, KID_ODOM_ASSOC, c->ring_w == 128 ? k_odom_assoc<128> : k_odom_assoc<64>, dim3((slots + 7) / 8, nb), dim3(256), 0, 1, it > 0, aa, op, sharp_slots);
    launch_lm_batch(c, slots > 0, la, nb, lp, 0, (integrate && last_it) ? 1 : 0, c->cfg.distortion != 0, false);   // local: cannot fail
  }
}

// restores the main stream on every exit of a function that re-points c->stream at the side streams
struct StreamGuard {
  aloam_ctx* c; cudaStream_t main;
  explicit StreamGuard(aloam_ctx* ctx) : c(ctx), main(ctx->stream) {}
  ~StreamGuard() { c->stream = main; }
};

void sync_all_streams(aloam_ctx* c) {
  cudaStream_t ss[] = {c->stream, c->s_ext, c->s_exa, c->s_idx, c->s_h2d, c->s_map};
  for (cudaStream_t s : ss) if (s) cudaStreamSynchronize(s);
}

}  // namespace

// The search index over the "last" clouds of feature set `slot` of lane `lane` (n_ls / n_lf points, their counts already queued on
// c->stream), then the check of every point's ring against the break tables just built (k_ring_offsets).  Synchronises;
// ALOAM_ERR_NOT_RING_MAJOR when a cloud is not ring-major.  aloam_odometry_set_last and aloam_lane_restore.
int index_last_clouds(aloam_ctx* c, int lane, int slot, int n_ls, int n_lf) {
  FeatBuf& f = c->lanes[lane].feat[slot];
  CUDA_CHECK_RET(cudaMemsetAsync(c->d_err, 0, 4, c->stream));
  run_grid_build(c, 1, &lane, slot, n_ls, n_lf);
  const auto ring_offsets = c->ring_w == 128 ? k_ring_offsets<128> : k_ring_offsets<64>;   // int(intensity) in 0 .. ring_w - 1
  if (n_ls > 0) LAUNCH(c, KID_RING_OFFSETS, ring_offsets, (n_ls + 255) / 256, 256, 0, f.less_sharp, n_ls, f.g_ls.fwd_end, c->d_err);
  if (n_lf > 0) LAUNCH(c, KID_RING_OFFSETS, ring_offsets, (n_lf + 255) / 256, 256, 0, f.less_flat, n_lf, f.g_lf.fwd_end, c->d_err);
  CUDA_CHECK_RET(cudaMemcpyAsync(&c->pin->ring_err, c->d_err, 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return c->pin->ring_err ? ALOAM_ERR_NOT_RING_MAJOR : ALOAM_OK;
}

extern "C" {

// ------------------------------------------------------------------------------------------------ feature extraction
int aloam_extract_features(aloam_ctx* c, aloam_cloud_view raw, aloam_cloud_view* full, aloam_cloud_view* sharp,
                           aloam_cloud_view* less_sharp, aloam_cloud_view* flat, aloam_cloud_view* less_flat) {
  if (!c || !full || !sharp || !less_sharp || !flat || !less_flat) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(raw);
  if (rc) return rc;
  if (raw.n == 0) return ALOAM_ERR_EMPTY_CLOUD;
  if (raw.n > c->max_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  Lane& L = c->lanes[0];
  CUDA_CHECK_RET(cudaMemcpyAsync(L.d_raw[0], raw.data, (size_t)raw.n * raw.stride_floats * 4, cudaMemcpyHostToDevice, c->stream));
  FeatBuf& f = L.feat[kApiCur];
  const int slot = c->parity;
  rc = run_features(c, L.d_raw[0], raw.n, raw.stride_floats, kApiCur);
  if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->feat_counts, f.counts, 16, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_sc, L.d_sc + slot, sizeof(ScanScalars), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (c->h_sc->error) {
    int e = c->h_sc->error;
    CUDA_CHECK_RET(cudaMemset(&(L.d_sc + slot)->error, 0, 4));
    return e;
  }
  const int n_full = c->h_sc->n_full;
  c->last_n_full = n_full;
  if (c->h_sc->first_valid == INT32_MAX) return ALOAM_ERR_EMPTY_CLOUD;
  const int* fc = c->pin->feat_counts;
  const int n[5] = {n_full, fc[0], fc[1], fc[2], fc[3]};
  const Pt4* src[5] = {L.d_full[0], f.sharp, f.less_sharp, f.flat, f.less_flat};
  for (int k = 0; k < 5; ++k)
    if (n[k] > 0) CUDA_CHECK_RET(cudaMemcpyAsync(c->h_out[k], src[k], (size_t)n[k] * 16, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  aloam_cloud_view* outs[5] = {full, sharp, less_sharp, flat, less_flat};
  for (int k = 0; k < 5; ++k) { outs[k]->data = reinterpret_cast<const float*>(c->h_out[k]); outs[k]->n = n[k]; outs[k]->stride_floats = 4; }
  return ALOAM_OK;
}

int aloam_debug_features(aloam_ctx* c, float* curvature, int* label, int* scan_start, int* scan_end) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const int n = c->last_n_full;
  if (curvature && n > 0) CUDA_CHECK_RET(cudaMemcpy(curvature, c->d_curv, (size_t)n * 4, cudaMemcpyDeviceToHost));
  if (label && n > 0) {
    std::vector<int8_t> tmp(n);
    CUDA_CHECK_RET(cudaMemcpy(tmp.data(), c->d_label, (size_t)n, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) label[i] = tmp[i];
  }
  if (scan_start) CUDA_CHECK_RET(cudaMemcpy(scan_start, c->lanes[0].d_scan_start, (size_t)c->cfg.n_scans * 4, cudaMemcpyDeviceToHost));
  if (scan_end) CUDA_CHECK_RET(cudaMemcpy(scan_end, c->lanes[0].d_scan_end, (size_t)c->cfg.n_scans * 4, cudaMemcpyDeviceToHost));
  return ALOAM_OK;
}

// ------------------------------------------------------------------------------------------------ odometry (API path)
int aloam_odometry_set_last(aloam_ctx* c, aloam_cloud_view corner_last, aloam_cloud_view surf_last) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_last); if (rc) return rc;
  rc = check_view(surf_last); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  FeatBuf& f = c->lanes[0].feat[kApiLast];
  rc = upload_cloud(c, corner_last, f.less_sharp, c->max_points); if (rc) return rc;
  rc = upload_cloud(c, surf_last, f.less_flat, c->max_points); if (rc) return rc;
  int* lc = c->pin->last_counts;
  lc[0] = 0; lc[1] = corner_last.n; lc[2] = 0; lc[3] = surf_last.n;
  CUDA_CHECK_RET(cudaMemcpyAsync(f.counts, lc, 16, cudaMemcpyHostToDevice, c->stream));
  rc = index_last_clouds(c, 0, kApiLast, corner_last.n, surf_last.n);
  if (rc) return rc;
  c->have_last = true;
  return ALOAM_OK;
}

static int upload_queries(aloam_ctx* c, aloam_cloud_view sharp, aloam_cloud_view flat, FeatBuf& f) {
  int rc = check_view(sharp); if (rc) return rc;
  rc = check_view(flat); if (rc) return rc;
  rc = upload_cloud(c, sharp, f.sharp, kMaxQueries); if (rc) return rc;
  rc = upload_cloud(c, flat, f.flat, kMaxQueries); if (rc) return rc;
  int* qc = c->pin->query_counts;
  qc[0] = sharp.n; qc[1] = 0; qc[2] = flat.n; qc[3] = 0;
  CUDA_CHECK_RET(cudaMemcpyAsync(f.counts, qc, 16, cudaMemcpyHostToDevice, c->stream));
  return ALOAM_OK;
}

int aloam_odometry_register(aloam_ctx* c, aloam_cloud_view sharp, aloam_cloud_view flat, double q[4], double t[3],
                            aloam_stats* stats) {
  if (!c || !q || !t) return ALOAM_ERR_INVALID_ARG;
  if (!c->have_last) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  Lane& L = c->lanes[0];
  int rc = upload_queries(c, sharp, flat, L.feat[kApiCur]); if (rc) return rc;
  for (int k = 0; k < 4; ++k) c->pin->pose_in[k] = q[k];
  for (int k = 0; k < 3; ++k) c->pin->pose_in[4 + k] = t[k];
  CUDA_CHECK_RET(cudaEventRecord(c->ev0, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_api_pose, c->pin->pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  run_register(c, 1, kLane0, kApiCur, kApiLast, sharp.n, flat.n, false, false, nullptr, c->d_api_pose);
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->pose_out, c->d_api_pose, 56, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, L.d_summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaEventRecord(c->ev1, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  for (int k = 0; k < 4; ++k) q[k] = c->pin->pose_out[k];
  for (int k = 0; k < 3; ++k) t[k] = c->pin->pose_out[4 + k];
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  fill_stats(c, stats, c->cfg.outer_iters, 0, ms);
  return ALOAM_OK;
}

int aloam_odometry_associate(aloam_ctx* c, aloam_cloud_view sharp, aloam_cloud_view flat, const double q[4], const double t[3],
                             int* corner_corr, int* plane_corr) {
  if (!c || !q || !t) return ALOAM_ERR_INVALID_ARG;
  if (!c->have_last) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  Lane& L = c->lanes[0];
  FeatBuf& cur = L.feat[kApiCur];
  int rc = upload_queries(c, sharp, flat, cur); if (rc) return rc;
  for (int k = 0; k < 4; ++k) c->pin->pose_in[k] = q[k];
  for (int k = 0; k < 3; ++k) c->pin->pose_in[4 + k] = t[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_api_pose, c->pin->pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  OdomParams op{c->cfg.dist_sq_thresh, c->cfg.nearby_scan, c->cfg.distortion};
  const int slots = sharp.n + flat.n;
  if (slots > 0) {
    Batch<AssocArgs> aa = {};
    aa.a[0] = AssocArgs{cur.sharp, cur.flat, cur.counts, last_corner(L.feat[kApiLast]), last_surf(L.feat[kApiLast]), c->d_api_pose, L.d_blocks, L.d_corr};
    LAUNCH(c, KID_ODOM_ASSOC, (c->ring_w == 128 ? k_odom_assoc<128> : k_odom_assoc<64>), dim3((slots + 7) / 8, 1), 256, 0, aa, op, sharp.n);
  }
  std::vector<int> h((size_t)slots * 4 + 4);
  if (slots > 0) CUDA_CHECK_RET(cudaMemcpyAsync(h.data(), L.d_corr, (size_t)slots * 16, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  for (int i = 0; i < sharp.n && corner_corr; ++i) { corner_corr[3 * i] = h[4 * i]; corner_corr[3 * i + 1] = h[4 * i + 1]; corner_corr[3 * i + 2] = h[4 * i + 3]; }
  for (int i = 0; i < flat.n && plane_corr; ++i) {
    const int* s = &h[4 * (size_t)(sharp.n + i)];
    plane_corr[4 * i] = s[0]; plane_corr[4 * i + 1] = s[1]; plane_corr[4 * i + 2] = s[2]; plane_corr[4 * i + 3] = s[3];
  }
  return ALOAM_OK;
}

// ------------------------------------------------------------------------------------------------ fused pipeline
static int scan_to_pose_impl(aloam_ctx* c, const float* d_raw, int n, int stride, double q_w[4], double t_w[3], aloam_stats* stats) {
  Lane& L = c->lanes[0];
  const int cur = c->frame % kFeatSlots, last = (c->frame + kFeatSlots - 1) % kFeatSlots;
  const int slot = c->parity;
  int rc = run_features(c, d_raw, n, stride, cur);
  if (rc) return rc;
  int flags = 0;
  // The search index over this scan's less-sharp / less-flat clouds (what replaces the kd-tree rebuild, laserOdometry.cpp:567-568)
  // is needed by the NEXT scan only: it is built on the index stream while this scan's association + LM run on the main stream, and
  // the call returns the pose without waiting for it (the next call, or aloam_scan_stream, waits on ev_idx).
  {
    StreamGuard guard(c);
    CUDA_CHECK_RET(cudaEventRecord(c->ev_feat[cur], c->stream));
    CUDA_CHECK_RET(cudaStreamWaitEvent(c->s_idx, c->ev_feat[cur], 0));
    if (!c->prof_on) c->stream = c->s_idx;   // (the per-kernel profiler times everything on one stream)
    run_grid_build(c, 1, kLane0, cur, c->less_sharp_upper(), std::min(n, c->max_points));
    CUDA_CHECK_RET(cudaEventRecord(c->ev_idx[cur], c->stream));
  }
  if (c->frame == 0) {
    flags |= ALOAM_FLAG_INITIALISED_ONLY;  // laserOdometry.cpp:267-271
  } else {
    CUDA_CHECK_RET(cudaStreamWaitEvent(c->stream, c->ev_idx[last], 0));   // the previous scan's index (built during the previous call)
    run_register(c, 1, kLane0, cur, last, c->fused_sharp_slots(), c->fused_flat_slots(), true, false, nullptr, nullptr);
  }
  CUDA_CHECK_RET(cudaEventRecord(c->ev_odo[cur], c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->world, L.d_world, 56, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, L.d_summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_sc, L.d_sc + slot, sizeof(ScanScalars), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaEventRecord(c->ev1, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  if (c->h_sc->error) {
    int e = c->h_sc->error;
    CUDA_CHECK_RET(cudaMemset(&(L.d_sc + slot)->error, 0, 4));
    return e;
  }
  if (c->h_sc->first_valid == INT32_MAX) return ALOAM_ERR_EMPTY_CLOUD;
  c->last_n_full = c->h_sc->n_full;
  for (int k = 0; k < 4; ++k) q_w[k] = c->pin->world[k];
  for (int k = 0; k < 3; ++k) t_w[k] = c->pin->world[4 + k];
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  if (c->frame == 0) { if (stats) { std::memset(stats, 0, sizeof(*stats)); stats->flags = flags; stats->ms_total = ms; } }
  else fill_stats(c, stats, c->cfg.outer_iters, flags, ms);
  c->frame++;
  return ALOAM_OK;
}

int aloam_scan_to_pose(aloam_ctx* c, aloam_cloud_view raw, double q_w[4], double t_w[3], aloam_stats* stats) {
  if (!c || !q_w || !t_w) return ALOAM_ERR_INVALID_ARG;
  if (c->lanes_mode) return ALOAM_ERR_STATE;   // the frame counter belongs to the lane schedule until aloam_reset_odometry
  int rc = check_view(raw); if (rc) return rc;
  if (raw.n == 0) return ALOAM_ERR_EMPTY_CLOUD;
  if (raw.n > c->max_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaEventRecord(c->ev0, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->lanes[0].d_raw[0], raw.data, (size_t)raw.n * raw.stride_floats * 4, cudaMemcpyHostToDevice, c->stream));
  return scan_to_pose_impl(c, c->lanes[0].d_raw[0], raw.n, raw.stride_floats, q_w, t_w, stats);
}

int aloam_scan_to_pose_device(aloam_ctx* c, const float* d_raw, int n, double q_w[4], double t_w[3], aloam_stats* stats) {
  if (!c || !q_w || !t_w || !d_raw) return ALOAM_ERR_INVALID_ARG;
  if (c->lanes_mode) return ALOAM_ERR_STATE;
  if (n <= 0) return ALOAM_ERR_EMPTY_CLOUD;
  if (n > c->max_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaEventRecord(c->ev0, c->stream));
  return scan_to_pose_impl(c, d_raw, n, 4, q_w, t_w, stats);
}

// Appends the next row to *t, `op` on the lane whose schedule state is *s (its raw scan v), and applies the op to *s: a START
// begins a trajectory at scan 0 -- in a mapped call (map) a mapped one that consumes the lane's arming, so that it localises or
// maps on a copy of the prior map --, a SCAN continues it, an IDLE ends it.  The one place a lane's scan index advances.
static void add_row(const aloam_ctx* c, StreamTable* t, LaneSched* s, int op, const aloam_cloud_view& v, bool map) {
  StreamRow r{op, -1, false, false, false, t->reg_total};
  if (op == ALOAM_LANE_IDLE) {
    s->running = false;
  } else {
    if (op == ALOAM_LANE_START) {
      s->running = true; s->mapped = map; s->scan = 0;
      s->localising = map && s->arm == ARM_LOCALISE;
      r.seed = map && s->arm == ARM_MAP_ON_PRIOR;
      if (map) s->arm = ARM_NONE;
    }
    r.scan = s->scan++;
    r.mapped = map && r.scan % c->cfg.mapping_skip_frame == 0;   // laserOdometry.cpp:570
    r.localise = map && s->localising;
    if (r.mapped) t->reg_total += v.n;
  }
  t->rows.push_back(r);
}

// What a stream call issues beside its odometry, fixed for the whole call from the context's settings
struct StreamSwitches {
  bool map;            // a mapped call: scan-to-map on s_map
  // registered clouds (aloam_set_registered_sink): every mapped row's ring-major cloud is stashed with its feature slot by stage C
  // and moved into the world by k_register_full after the row's mapper frame; without a sink none of this is issued
  bool sink;
  // per-row records (aloam_set_map_rows): k_map_rows after every frame, the tracking score after every localising frame when scoring is
  // on; without recording none of this is issued
  bool rec, score;
  bool recov;          // recovery of localising lanes (aloam_set_recovery, recover.cu): four more launches after every scored localising frame
  bool place;          // keyframes (aloam_set_place, place.cu): three more launches after every mapping frame, one copy of the place rows
  bool loop;           // loop verification (aloam_set_loops, loop.cu): keyframe clouds after every mapping frame and the verification of
                       // its triggered rows, one copy of the loop rows
  bool reset_stores;   // a START also resets its lane's cube store
  StreamSwitches(const aloam_ctx* c, bool mapped, bool reset)
      : map(mapped), sink(map && c->reg_sink), rec(map && c->rows_on), score(rec && c->rows_max_score > 0), recov(score && c->rec_on),
        place(map && c->place_on), loop(place && c->loop_on), reset_stores(reset) {}
};
#define STREAM_TRY(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { fprintf(stderr, "[aloam_b200] CUDA error %s at %s:%d\n", cudaGetErrorName(_e), __FILE__, __LINE__); return ALOAM_ERR_CUDA; } } while (0)

// ---- scan-to-map of one step on s_map (laserMapping.cpp process()): the scan's less-sharp / less-flat clouds and its odometry pose
//      go to the mapping stage on the device -- what the reference ships through /laser_cloud_corner_last, /laser_cloud_surf_last
//      and /laser_odom_to_init (laserOdometry.cpp:570-591 -> laserMapping.cpp:278-288) never leaves HBM.
//      One frame covers every mapped lane of the step: each launch of it serves all of them, each with its own cube store; the
//      step's mapped lanes that localise go to one locate frame against the prior map instead (no cube store).  Scan j of a
//      trajectory is mapped when j % mapping_skip_frame == 0 (laserOdometry.cpp:570); the others get the high-frequency pose of
//      laserMapping.cpp:197-229 from one k_mapper_high_freq launch.  A step that maps no lane issues no frame and does not record
//      ev_mapdone[cur], so the next writer of this feature slot (stage C, four steps on) waits only on a frame that read it.
// The step's rows are row[0 .. nb-1], rows r0 .. r0+nb-1 of the call; act[0 .. na-1] its non-idle lanes, cur its feature slot and
// nmax its largest scan.  Leaves c->stream on s_map; returns the error the call fails with.
static int map_stage(aloam_ctx* c, const StreamSwitches& w, const StreamRow* row, size_t r0, const int* act, int na, int cur, int nmax) {
  STREAM_TRY(cudaStreamWaitEvent(c->s_map, c->ev_odo[cur], 0));
  c->stream = c->s_map;
  MapperIn fr[3][ALOAM_MAX_BATCH];   // the records of the mapping frame, of the locate frame and of the high-frequency poses
  int n_fr[3] = {0, 0, 0};
  for (int i = 0; i < na; ++i) {
    const int l = act[i];
    const FeatBuf& fc = c->lanes[l].feat[cur]; const size_t slot = (r0 + l) * 7;
    const int g = !row[l].mapped ? 2 : row[l].localise;
    fr[g][n_fr[g]++] = MapperIn{fc.less_sharp, fc.counts + 1, fc.less_flat, fc.counts + 3, c->d_poses + slot, c->d_map_poses + slot, l,
                                w.reset_stores && row[l].op == ALOAM_LANE_START && !row[l].seed, row[l].localise, row[l].seed};
  }
  const int n_upper_c = c->less_sharp_upper(), n_upper_s = std::min(nmax, c->max_points);
  for (int loc = 0; loc < 2; ++loc) {   // the mapping frame, then the locate frame, each followed by its rows and registered clouds
    const MapperIn* in = fr[loc]; const int n = n_fr[loc];
    if (n == 0) continue;
    MapRowRec* rows[ALOAM_MAX_BATCH] = {};                    // the row slots of the frame's records
    const Pt4* src[ALOAM_MAX_BATCH] = {}; const int* nf[ALOAM_MAX_BATCH] = {}; Pt4* dst[ALOAM_MAX_BATCH] = {};   // their registered clouds
    LaneFrame* lp[ALOAM_MAX_BATCH] = {}; const double* init[ALOAM_MAX_BATCH] = {};                                    // their locators
    for (int j = 0; j < n; ++j) {
      Lane& L = c->lanes[in[j].lane];
      if (w.rec) rows[j] = c->d_rows + r0 + in[j].lane;
      if (w.sink) { src[j] = L.feat[cur].full; nf[j] = c->d_scan_nfull + r0 + in[j].lane; dst[j] = c->reg_sink + row[in[j].lane].reg_begin; }
      lp[j] = L.locator; init[j] = L.init;
    }
    int rc = loc ? locate_step_device(c, n, in, lp, init, n_upper_c, n_upper_s) : mapper_step_device(c, n, in, n_upper_c, n_upper_s);
    if (rc) return rc;
    if (w.rec) { rc = map_rows_device(c, n, in, rows, loc ? c->rows_max_score : 0); if (rc) return rc; }
    if (loc && w.score) { rc = track_score_device(c, n, in, rows, n_upper_c, n_upper_s); if (rc) return rc; }
    if (loc && w.recov) { rc = recover_device(c, n, in, rows); if (rc) return rc; }
    if (!loc && w.place) {   // keyframes of the mapping frame's rows, from their refined map poses
      int scan[ALOAM_MAX_BATCH]; bool start[ALOAM_MAX_BATCH]; aloam_place_row* prow[ALOAM_MAX_BATCH];
      for (int j = 0; j < n; ++j) {
        const StreamRow& R = row[in[j].lane];
        scan[j] = R.scan; start[j] = R.op == ALOAM_LANE_START; prow[j] = place_rows_device(c) + r0 + in[j].lane;
      }
      int n_upper = 0;
      rc = place_record_device(c, n, in, scan, start, prow, &n_upper); if (rc) return rc;
      if (w.loop) { rc = loop_record_device(c, n, in, prow, r0, n_upper); if (rc) return rc; }
    }
    for (int j = 0; loc && j < n; ++j) c->lanes[in[j].lane].window = true;
    // /velodyne_cloud_registered of the frame's rows, before the lanes' next frame replaces the refined pose
    if (w.sink) { rc = mapper_register_full_device(c, n, in, src, nf, dst, nmax); if (rc) return rc; }
  }
  if (n_fr[0] + n_fr[1] > 0) STREAM_TRY(cudaEventRecord(c->ev_mapdone[cur], c->s_map));
  return n_fr[2] > 0 ? mapper_high_freq_device(c, n_fr[2], fr[2]) : ALOAM_OK;
}

// Issues every step of a stream call on the rows t, drains it and checks what its scans left on the device (scan_stream_run);
// last_op: the last non-idle op of every lane in this call (IDLE: none).  Returns the error the call fails with.
static int stream_issue(aloam_ctx* c, const aloam_cloud_view* raws, const StreamTable& t, int n_scans, int nb, int device_resident,
                        const StreamSwitches& w, int* last_op) {
  const cudaStream_t s_main = c->stream;
  const auto host_t0 = std::chrono::steady_clock::now();
  if (w.map) {
    for (int l = 0; l < nb; ++l)   // every frame's error bits of this call (a lane that only localises has no cube store)
      for (int loc = 0; loc < 2; ++loc)
        if (const LaneFrame* f = lane_frame(c, l, loc)) STREAM_TRY(cudaMemsetAsync(frame_view(f).err_acc, 0, sizeof(int), s_main));
    const int rc = peer_err_reset(c); if (rc) return rc;
  }
  STREAM_TRY(cudaEventRecord(c->ev0, s_main));
  // everything issued on the main stream before this call (reset, earlier calls) is ordered before the side streams.
  // Waiting on an event that was never recorded, or whose work finished in an earlier call, is a no-op -- so the
  // per-scan waits below need no "first iterations" special cases.
  for (cudaStream_t s : {c->s_h2d, c->s_exa, c->s_ext, c->s_idx, c->s_map}) STREAM_TRY(cudaStreamWaitEvent(s, c->ev0, 0));
  const float* d_raw[ALOAM_MAX_BATCH];      // per record
  int ns[ALOAM_MAX_BATCH];
  int act[ALOAM_MAX_BATCH], scanning[ALOAM_MAX_BATCH], starting[ALOAM_MAX_BATCH];   // lanes of the step: all, registering, initialising
  int issued = 0;
  for (int k = 0; k < n_scans; ++k) {
    const StreamRow* row = t.rows.data() + (size_t)k * nb;   // the step's rows, one per lane
    // a lane's first scan, its START, only initialises (laserOdometry.cpp:267-271)
    int na = 0, n_scan = 0, n_start = 0;
    for (int l = 0; l < nb; ++l) {
      if (row[l].op == ALOAM_LANE_IDLE) continue;
      act[na++] = l; last_op[l] = row[l].op;
      if (row[l].op == ALOAM_LANE_START) starting[n_start++] = l; else scanning[n_scan++] = l;
    }
    if (na == 0) continue;                  // an all-idle step: nothing to run, the frame does not advance
    const int f = c->frame;                 // global frame number of this step
    const int b = issued++ & 1;             // raw / ring-major double buffer
    const int cur = f % kFeatSlots, last = (f + kFeatSlots - 1) % kFeatSlots;
    const aloam_cloud_view* rv = raws + (size_t)k * nb;
    int nmax = 0;
    for (int i = 0; i < na; ++i) { ns[i] = rv[act[i]].n; nmax = std::max(nmax, ns[i]); }
    if (device_resident) {
      for (int i = 0; i < na; ++i) d_raw[i] = rv[act[i]].data;
    } else {
      STREAM_TRY(cudaStreamWaitEvent(c->s_h2d, c->ev_rawfree[b], 0));   // stage A of scan k-2 has consumed the buffers
      for (int i = 0; i < na; ++i) {
        const int l = act[i];
        STREAM_TRY(cudaMemcpyAsync(c->lanes[l].d_raw[b], rv[l].data, (size_t)rv[l].n * rv[l].stride_floats * 4, cudaMemcpyHostToDevice, c->s_h2d));
        d_raw[i] = c->lanes[l].d_raw[b];
      }
      STREAM_TRY(cudaEventRecord(c->ev_h2d[b], c->s_h2d));
      STREAM_TRY(cudaStreamWaitEvent(c->s_exa, c->ev_h2d[b], 0));
    }
    // ---- stage A (ring binning) on s_exa: needs full[b] free, i.e. stage B of scan k-2 done
    STREAM_TRY(cudaStreamWaitEvent(c->s_exa, c->ev_b[b], 0));
    // with a sink, full[b] is also read by the stash copy of stage C (which waits on the mapper frame four steps back)
    if (w.sink) STREAM_TRY(cudaStreamWaitEvent(c->s_exa, c->ev_stash[b], 0));
    c->stream = c->s_exa;
    // A START re-arms the lane's ScanScalars slot (k_ring_scan arms it only for a lane that ran the step before) and, below, resets its pose.
    // At a lockstep call's first step these copies change nothing: k_ring_scan armed the slot with d_sc_init's four fields, start_ori /
    // end_ori are written (k_classify, k_ring_scan) before they are read, and aloam_reset_odometry has put the identity in d_pose / d_world.
    for (int i = 0; i < n_start; ++i)
      STREAM_TRY(cudaMemcpyAsync(c->lanes[starting[i]].d_sc + c->parity, c->d_sc_init, sizeof(ScanScalars), cudaMemcpyDeviceToDevice, c->s_exa));
    int sc_slot = 0;
    int rc = run_features_a(c, na, act, d_raw, ns, device_resident ? 4 : rv[act[0]].stride_floats, b, &sc_slot, c->d_scan_nfull + (size_t)k * nb);
    if (rc) return rc;
    if (!device_resident) STREAM_TRY(cudaEventRecord(c->ev_rawfree[b], c->s_exa));
    STREAM_TRY(cudaEventRecord(c->ev_a[b], c->s_exa));
    // ---- stage B (k_ring_features, the longest kernel) on s_ext: needs stage A of this scan and the staging set b free
    //      (its previous content was consumed by the compaction of scan k-2)
    c->stream = c->s_ext;
    STREAM_TRY(cudaStreamWaitEvent(c->s_ext, c->ev_a[b], 0));
    STREAM_TRY(cudaStreamWaitEvent(c->s_ext, c->ev_cmp[b], 0));
    rc = run_features_b1(c, na, act, b, sc_slot);
    if (rc) return rc;
    STREAM_TRY(cudaEventRecord(c->ev_b[b], c->s_ext));
    // ---- stage C on s_idx: ring-ordered compaction into feat[f % kFeatSlots] -- that slot was last read by the odometry
    //      of frame f - (kFeatSlots - 1) as its "last" clouds -- then the search index over its less-sharp / less-flat
    //      clouds, which only the NEXT scan's odometry needs
    c->stream = c->s_idx;
    STREAM_TRY(cudaStreamWaitEvent(c->s_idx, c->ev_b[b], 0));
    STREAM_TRY(cudaStreamWaitEvent(c->s_idx, c->ev_odo[(f + 1) % kFeatSlots], 0));
    STREAM_TRY(cudaStreamWaitEvent(c->s_idx, c->ev_mapdone[cur], 0));   // the last mapper frame that read this slot (of frame f - kFeatSlots at the latest) is done
    if (w.sink) {   // the ring-major cloud of every mapped row goes with the slot until its mapper frame has registered it
      for (int i = 0; i < na; ++i)
        if (row[act[i]].mapped) { Lane& L = c->lanes[act[i]]; STREAM_TRY(cudaMemcpyAsync(L.feat[cur].full, L.d_full[b], (size_t)ns[i] * sizeof(Pt4), cudaMemcpyDeviceToDevice, c->s_idx)); }
      STREAM_TRY(cudaEventRecord(c->ev_stash[b], c->s_idx));
    }
    rc = run_features_b2(c, na, act, b, cur, false);
    if (rc) return rc;
    STREAM_TRY(cudaEventRecord(c->ev_cmp[b], c->s_idx));
    STREAM_TRY(cudaEventRecord(c->ev_feat[cur], c->s_idx));
    run_grid_build(c, na, act, cur, c->less_sharp_upper(), std::min(nmax, c->max_points));
    STREAM_TRY(cudaEventRecord(c->ev_idx[cur], c->s_idx));
    c->stream = s_main;
    // ---- association + LM on the main stream: this scan's sharp / flat points, the previous scan's clouds + index
    STREAM_TRY(cudaStreamWaitEvent(s_main, c->ev_feat[cur], 0));
    STREAM_TRY(cudaStreamWaitEvent(s_main, c->ev_idx[last], 0));
    // the last solve of the scan writes the integrated world pose into its slot of d_poses (no copy on the critical chain)
    double* slots = c->d_poses + (size_t)k * nb * 7;
    for (int i = 0; i < n_start; ++i) {   // a new trajectory: warm start and world pose back to the identity, in stream order
      Lane& L = c->lanes[starting[i]];
      STREAM_TRY(cudaMemcpyAsync(L.d_pose, c->d_ident, 56, cudaMemcpyDeviceToDevice, s_main));
      STREAM_TRY(cudaMemcpyAsync(L.d_world, c->d_ident, 56, cudaMemcpyDeviceToDevice, s_main));
      STREAM_TRY(cudaMemcpyAsync(slots + (size_t)starting[i] * 7, L.d_world, 56, cudaMemcpyDeviceToDevice, s_main));
    }
    if (n_scan > 0) run_register(c, n_scan, scanning, cur, last, c->fused_sharp_slots(), c->fused_flat_slots(), true, false, slots, nullptr);
    STREAM_TRY(cudaEventRecord(c->ev_odo[cur], s_main));
    if (w.map) {
      rc = map_stage(c, w, row, (size_t)k * nb, act, na, cur, nmax);
      if (rc) return rc;
      c->stream = s_main;
    }
    c->frame++;
  }
  if (getenv("ALOAM_DEBUG_TIMING")) fprintf(stderr, "[aloam_b200] scan_stream: host issued %d x %d scans in %.1f us (%.1f us / step)\n", n_scans, nb,
      std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - host_t0).count(),
      std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - host_t0).count() / n_scans);
  const size_t total = (size_t)n_scans * nb;
  STREAM_TRY(cudaMemcpyAsync(c->h_poses, c->d_poses, total * 56, cudaMemcpyDeviceToHost, s_main));
  if (w.map) {
    STREAM_TRY(cudaEventRecord(c->ev_mapend, c->s_map));   // the last mapper frame and the last high-frequency poses
    STREAM_TRY(cudaStreamWaitEvent(s_main, c->ev_mapend, 0));
    STREAM_TRY(cudaMemcpyAsync(c->h_poses + (size_t)kMaxStreamScans * 7, c->d_map_poses, total * 56, cudaMemcpyDeviceToHost, s_main));
    if (w.rec) STREAM_TRY(cudaMemcpyAsync(c->h_rows, c->d_rows, total * sizeof(MapRowRec), cudaMemcpyDeviceToHost, s_main));
    if (w.place) STREAM_TRY(cudaMemcpyAsync(place_rows_host(c), place_rows_device(c), total * sizeof(aloam_place_row), cudaMemcpyDeviceToHost, s_main));
    if (w.loop) STREAM_TRY(cudaMemcpyAsync(loop_rows_host(c), loop_rows_device(c), total * loop_row_bytes(), cudaMemcpyDeviceToHost, s_main));
    for (int l = 0; l < nb; ++l) {
      int* dst[2] = {&c->pin->mapper_err_lane[l], &c->pin->locate_err_lane[l]};
      *dst[0] = *dst[1] = 0;
      for (int loc = 0; loc < 2; ++loc)
        if (const LaneFrame* f = lane_frame(c, l, loc)) STREAM_TRY(cudaMemcpyAsync(dst[loc], frame_view(f).err_acc, sizeof(int), cudaMemcpyDeviceToHost, s_main));
    }
    const int rc = peer_err_fetch(c, &c->pin->peer_err); if (rc) return rc;
  }
  for (int l = 0; l < nb; ++l) {
    STREAM_TRY(cudaMemcpyAsync(c->h_summary + 4 * l, c->lanes[l].d_summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, s_main));
    STREAM_TRY(cudaMemcpyAsync(c->h_sc + 3 * l, c->lanes[l].d_sc, 3 * sizeof(ScanScalars), cudaMemcpyDeviceToHost, s_main));
  }
  STREAM_TRY(cudaEventRecord(c->ev1, s_main));
  STREAM_TRY(cudaStreamSynchronize(s_main));
  // the ring-binning stream has produced every n_full by now (the odometry of the last scan depends on it)
  STREAM_TRY(cudaMemcpyAsync(c->h_scan_nfull, c->d_scan_nfull, total * 4, cudaMemcpyDeviceToHost, s_main));
  sync_all_streams(c);
  STREAM_TRY(cudaGetLastError());
  prof_collect(c);
  for (int l = 0; l < nb; ++l)
    for (int b = 0; b < 3; ++b)
      if (c->h_sc[3 * l + b].error) return c->h_sc[3 * l + b].error;
  for (size_t i = 0; i < total; ++i)   // (an idle entry has no scan)
    if (t.rows[i].op != ALOAM_LANE_IDLE && c->h_scan_nfull[i] <= 0) return ALOAM_ERR_EMPTY_CLOUD;   // scanRegistration.cpp:136-137 left nothing of this scan
  return ALOAM_OK;
}
#undef STREAM_TRY

// Pipelined form of aloam_scan_to_pose over `nb` lanes: ring binning of step k+1 (s_exa), per-ring extraction (s_ext), compaction
// + index build (s_idx) run concurrently with association + LM of step k (main stream) and the host->device copies of step k+2
// (s_h2d) -- the overlap the reference gets from its three ROS processes.  Every stream call runs this driver on the rows t of its
// lane schedule (scan-major as raws and poses: entry k * nb + b).  A step packs its non-idle lanes into records 0 .. na-1 of every launch
// (record i = lane act[i], which owns the buffers, pose slots and cube store); an all-idle step issues nothing.  reset_stores: a
// START also resets its lane's cube store.  The rows that localise register against the prior map in one locate frame per step,
// beside the mapping frame of the step's other lanes.  The caller has checked the views and the schedule, built its rows t and
// created the cube stores and locators.
static int scan_stream_run(aloam_ctx* c, const aloam_cloud_view* raws, StreamTable table, int n_scans, int nb, int device_resident, double* poses,
                           double* map_poses, aloam_stats* stats_last, bool reset_stores) {
  StreamGuard guard(c);
  const StreamSwitches w(c, map_poses != nullptr, reset_stores);
  MappedCall& M = c->last_mapped;
  if (w.map) {   // this call's rows replace the last mapped call's, unreadable until the call has drained
    M.table = std::move(table); M.n_scans = n_scans; M.nb = nb;
    M.registered = M.records = M.places = M.loops = false; M.recovered = w.recov;
    recover_call_done(c);   // no lane's candidate scores belong to this call yet
  }
  const StreamTable& t = w.map ? M.table : table;
  int last_op[ALOAM_MAX_BATCH] = {};
  if (const int rc = stream_issue(c, raws, t, n_scans, nb, device_resident, w, last_op)) {
    // drain everything, clear the sticky device errors and forget the odometry state: a partial pipeline cannot be rolled back
    sync_all_streams(c);
    cudaGetLastError();
    for (Lane& L : c->lanes) for (int b = 0; b < 3; ++b) cudaMemset(&(L.d_sc + b)->error, 0, 4);
    c->stream = guard.main;
    aloam_reset_odometry(c);
    return rc;
  }
  const size_t total = (size_t)n_scans * nb;
  std::memcpy(poses, c->h_poses, total * 56);
  if (map_poses) std::memcpy(map_poses, c->h_poses + (size_t)kMaxStreamScans * 7, total * 56);
  for (size_t i = 0; i < total; ++i)
    if (t.rows[i].op == ALOAM_LANE_IDLE)
      for (int j = 0; j < 7; ++j) { poses[i * 7 + j] = NAN; if (map_poses) map_poses[i * 7 + j] = NAN; }
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  if (stats_last) {
    for (int l = 0; l < nb; ++l) {
      if (last_op[l] == ALOAM_LANE_IDLE) std::memset(&stats_last[l], 0, sizeof(aloam_stats));   // idle all call
      else if (last_op[l] == ALOAM_LANE_START) { std::memset(&stats_last[l], 0, sizeof(aloam_stats)); stats_last[l].flags = ALOAM_FLAG_INITIALISED_ONLY; stats_last[l].ms_total = ms; }
      else fill_stats_from(c->h_summary + 4 * l, &stats_last[l], c->cfg.outer_iters, 0, ms);
    }
  }
  if (w.map) {   // the call's rows are readable (after ALOAM_ERR_CAPACITY and ALOAM_ERR_COMM below too: they name the row that was hit)
    M.reg_count.resize(total);
    for (size_t r = 0; r < total; ++r) M.reg_count[r] = w.sink && t.rows[r].mapped ? c->h_scan_nfull[r] : 0;
    M.registered = true; M.records = w.rec; M.places = w.place; M.loops = w.loop;
    recover_call_done(c);
    // as aloam_mapper_step: a voxel index range beyond the key width in any frame of any lane means its map results would be wrong
    c->pin->mapper_err = 0;
    for (int l = 0; l < nb; ++l) c->pin->mapper_err |= c->pin->mapper_err_lane[l] | c->pin->locate_err_lane[l];
    if (c->pin->mapper_err & 1) return ALOAM_ERR_CAPACITY;
    if (c->pin->peer_err) return ALOAM_ERR_COMM;   // a peer did not answer: a map pose rests on a partial sum
  }
  return ALOAM_OK;
}

static bool stream_args_ok(const aloam_ctx* c, const aloam_cloud_view* raws, int n_scans, int nb, const double* poses, const double* map_poses) {
  return c && raws && poses && n_scans >= 1 && nb >= 1 && nb <= c->n_lanes && (long long)n_scans * nb <= kMaxStreamScans && (!map_poses || c->cfg.max_map_points > 0);
}

// the lockstep calls: every lane STARTs at the context's first step, SCANs after it and keeps its cube store over a START
static int scan_stream_lockstep(aloam_ctx* c, const aloam_cloud_view* raws, int n_scans, int nb, int device_resident, double* poses,
                                double* map_poses, aloam_stats* stats_last) {
  if (!stream_args_ok(c, raws, n_scans, nb, poses, map_poses)) return ALOAM_ERR_INVALID_ARG;
  if (c->lanes_mode) return ALOAM_ERR_STATE;   // the frame counter belongs to the lane schedule until aloam_reset_odometry
  for (int k = 0; k < n_scans * nb; ++k) {
    int rc = check_view(raws[k]); if (rc) return rc;
    if (raws[k].n == 0) return ALOAM_ERR_EMPTY_CLOUD;
    if (raws[k].n > c->max_points) return ALOAM_ERR_CAPACITY;
    if (device_resident && raws[k].stride_floats != 4) return ALOAM_ERR_INVALID_ARG;
    if (raws[k].stride_floats != raws[k - k % nb].stride_floats) return ALOAM_ERR_INVALID_ARG;   // one stride per step
  }
  // the rows from the lanes' scan indices alone: a lockstep call neither localises nor changes a lane's mode or arming
  StreamTable t((size_t)n_scans * nb);
  LaneSched s[ALOAM_MAX_BATCH];
  for (int l = 0; l < nb; ++l) s[l].scan = c->lanes[l].sched.scan;
  for (int i = 0; i < n_scans * nb; ++i) add_row(c, &t, &s[i % nb], c->frame == 0 && i < nb ? ALOAM_LANE_START : ALOAM_LANE_SCAN, raws[i], map_poses);
  if (map_poses && c->reg_sink && t.reg_total > c->reg_cap) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  for (int l = 0; map_poses && l < nb; ++l) { int rc = mapper_ensure(c, l); if (rc) return rc; }   // creates the cube stores this call needs
  for (int l = 0; l < nb; ++l) c->lanes[l].sched.scan = s[l].scan;
  return scan_stream_run(c, raws, std::move(t), n_scans, nb, device_resident, poses, map_poses, stats_last, false);
}

int aloam_scan_stream(aloam_ctx* c, const aloam_cloud_view* raws, int n_scans, int device_resident, double* poses, aloam_stats* stats_last) {
  return scan_stream_lockstep(c, raws, n_scans, 1, device_resident, poses, nullptr, stats_last);
}

int aloam_scan_stream_mapped(aloam_ctx* c, const aloam_cloud_view* raws, int n_scans, int device_resident, double* odom_poses, double* map_poses,
                             aloam_stats* stats_last) {
  if (!map_poses) return ALOAM_ERR_INVALID_ARG;
  return scan_stream_lockstep(c, raws, n_scans, 1, device_resident, odom_poses, map_poses, stats_last);
}

int aloam_scan_stream_batch(aloam_ctx* c, const aloam_cloud_view* raws, int n_scans, int batch, int device_resident, double* poses,
                            aloam_stats* stats_last) {
  return scan_stream_lockstep(c, raws, n_scans, batch, device_resident, poses, nullptr, stats_last);
}

int aloam_scan_stream_mapped_batch(aloam_ctx* c, const aloam_cloud_view* raws, int n_scans, int batch, int device_resident, double* odom_poses,
                                   double* map_poses, aloam_stats* stats_last) {
  if (!map_poses) return ALOAM_ERR_INVALID_ARG;
  if (c && sharded_job(c)) return ALOAM_ERR_STATE;   // a sharded job maps one trajectory (aloam_scan_stream_mapped)
  return scan_stream_lockstep(c, raws, n_scans, batch, device_resident, odom_poses, map_poses, stats_last);
}

int aloam_scan_stream_lanes(aloam_ctx* c, const aloam_cloud_view* raws, const int* lane_ops, int n_scans, int batch, int device_resident,
                            double* odom_poses, double* map_poses, aloam_stats* stats_last) {
  if (!lane_ops) return ALOAM_ERR_INVALID_ARG;
  if (c && sharded_job(c)) return ALOAM_ERR_STATE;   // a sharded job maps one trajectory (aloam_scan_stream_mapped)
  if (!stream_args_ok(c, raws, n_scans, batch, odom_poses, map_poses)) return ALOAM_ERR_INVALID_ARG;
  // the whole schedule is checked on a copy of the lanes' schedule state before anything changes; lanes >= batch are idle all call
  const bool map = map_poses != nullptr;
  LaneSched s[ALOAM_MAX_BATCH];
  for (int l = 0; l < c->n_lanes; ++l) { s[l] = c->lanes[l].sched; s[l].running = s[l].running && l < batch; }
  bool maps[ALOAM_MAX_BATCH] = {}, localises[ALOAM_MAX_BATCH] = {};   // the lane has a mapping / a localising scan in this call
  bool seeds = false;                                                 // a START maps on a copy of the prior map
  for (size_t i = 0; i < (size_t)n_scans * batch; ++i)
    if (lane_ops[i] < ALOAM_LANE_IDLE || lane_ops[i] > ALOAM_LANE_START) return ALOAM_ERR_INVALID_ARG;
  StreamTable t((size_t)n_scans * batch);
  int run_err = ALOAM_OK;   // a scan that cannot run fails the call like a run-time error
  for (int k = 0; k < n_scans; ++k) {
    int stride = 0;
    for (int l = 0; l < batch; ++l) {
      const int op = lane_ops[(size_t)k * batch + l];
      const aloam_cloud_view& v = raws[(size_t)k * batch + l];
      if (op != ALOAM_LANE_IDLE) {   // an idle row's view is not read
        int rc = check_view(v); if (rc) return rc;
        if (v.n > 0) {
          if (device_resident && v.stride_floats != 4) return ALOAM_ERR_INVALID_ARG;
          if (stride && v.stride_floats != stride) return ALOAM_ERR_INVALID_ARG;   // one stride per step
          stride = v.stride_floats;
        }
        // a SCAN continues the trajectory its lane runs, in the mode (mapped or not) it was started in
        if (op == ALOAM_LANE_SCAN && (!s[l].running || s[l].mapped != map)) return ALOAM_ERR_STATE;
        if (!run_err && v.n == 0) run_err = ALOAM_ERR_EMPTY_CLOUD;
        if (!run_err && v.n > c->max_points) run_err = ALOAM_ERR_CAPACITY;
      }
      add_row(c, &t, &s[l], op, v, map);
      if (map && op != ALOAM_LANE_IDLE) (t.rows.back().localise ? localises : maps)[l] = true;
      seeds = seeds || t.rows.back().seed;
    }
  }
  if (map && c->reg_sink && t.reg_total > c->reg_cap) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (run_err) { if (map) c->last_mapped.records = c->last_mapped.places = c->last_mapped.loops = false; aloam_reset_odometry(c); return run_err; }
  for (int l = 0; map && l < batch; ++l) {   // creates the cube stores and locators this call needs: a lane that only localises gets no cube store
    int rc = localises[l] ? locator_ensure(c, l) : ALOAM_OK; if (rc) return rc;
    rc = maps[l] || !localises[l] ? mapper_ensure(c, l) : ALOAM_OK; if (rc) return rc;
  }
  if (seeds) { const int rc = mapper_seed_ensure(c); if (rc) return rc; }
  // committed before anything is issued: a later failure ends in aloam_reset_odometry, a key overflow leaves the lanes running
  c->lanes_mode = true;
  for (int l = 0; l < c->n_lanes; ++l) c->lanes[l].sched = s[l];
  return scan_stream_run(c, raws, std::move(t), n_scans, batch, device_resident, odom_poses, map_poses, stats_last, true);
}

int aloam_set_registered_sink(aloam_ctx* c, float* data, long long capacity) {
  if (!c || capacity < 0) return ALOAM_ERR_INVALID_ARG;
  if (!data) { c->reg_sink = nullptr; c->reg_cap = 0; return ALOAM_OK; }
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  cudaPointerAttributes at = {};
  if (cudaPointerGetAttributes(&at, data) != cudaSuccess) { cudaGetLastError(); return ALOAM_ERR_INVALID_ARG; }
  const bool device = (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == c->cfg.device;
  if (!(device || at.type == cudaMemoryTypeHost) || !at.devicePointer) return ALOAM_ERR_INVALID_ARG;   // pageable: no device address
  if (!c->ev_stash[1]) {   // first use: the stash of every lane, then the events (the last one marks the group as ready)
    for (Lane& L : c->lanes)
      for (int s = 0; s < kFeatSlots; ++s)
        if (!L.feat[s].full) CUDA_CHECK_RET(dalloc(c, &L.feat[s].full, (size_t)c->max_points));
    for (cudaEvent_t& e : c->ev_stash) if (!e) CUDA_CHECK_RET(ecreate(c, &e, cudaEventDisableTiming));
  }
  c->reg_sink = static_cast<Pt4*>(at.devicePointer);
  c->reg_cap = capacity;
  return ALOAM_OK;
}

int aloam_registered_rows(aloam_ctx* c, long long* begin, int* count, int rows) {
  if (!c || rows < 0 || (rows > 0 && (!begin || !count))) return ALOAM_ERR_INVALID_ARG;
  const MappedCall& M = c->last_mapped;
  if (const int rc = M.check(M.registered, rows)) return rc;
  for (int r = 0; r < rows; ++r) { begin[r] = M.table.rows[r].reg_begin; count[r] = M.reg_count[r]; }
  return ALOAM_OK;
}

// ------------------------------------------------------------------------------------------------ fine-grained
int aloam_knn(aloam_ctx* c, int which, aloam_cloud_view queries, int k, int* idx, float* sqdist) {
  if (!c || !idx || !sqdist || k < 1) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(queries); if (rc) return rc;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  if (which == 0 || which == 1) {
    if (!c->have_last) return ALOAM_ERR_STATE;
    if (k != 1) return ALOAM_ERR_INVALID_ARG;  // the reference only asks for k = 1 on these trees (laserOdometry.cpp:302,390)
    rc = upload_cloud(c, queries, c->d_query, c->max_points); if (rc) return rc;
    if (queries.n > 0) {
      const FeatBuf& f0 = c->lanes[0].feat[kApiLast];
      LastCloud L = which == 0 ? last_corner(f0) : last_surf(f0);
      LAUNCH(c, KID_KNN_LAST, (c->ring_w == 128 ? k_knn_last<128> : k_knn_last<64>), (queries.n + 7) / 8, 256, 0, L, c->d_query, queries.n, c->d_knn_idx, c->d_knn_d);
      CUDA_CHECK_RET(cudaMemcpyAsync(idx, c->d_knn_idx, (size_t)queries.n * 4, cudaMemcpyDeviceToHost, c->stream));
      CUDA_CHECK_RET(cudaMemcpyAsync(sqdist, c->d_knn_d, (size_t)queries.n * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
    CUDA_CHECK_RET(cudaGetLastError());
    return ALOAM_OK;
  }
  if (which == 2 || which == 3) return aloam_map_knn_impl(c, which, queries, k, idx, sqdist);
  return ALOAM_ERR_INVALID_ARG;
}

int aloam_transform_to_end(aloam_ctx* c, aloam_cloud_view in, const double q[4], const double t[3], int distortion, aloam_cloud_view* out) {
  if (!c || !q || !t || !out) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(in); if (rc) return rc;
  if (in.n > c->max_points) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  out->data = reinterpret_cast<const float*>(c->h_out[0]); out->n = in.n; out->stride_floats = 4;
  if (in.n == 0) return ALOAM_OK;
  rc = upload_cloud(c, in, c->d_query, c->max_points); if (rc) return rc;
  for (int k = 0; k < 4; ++k) c->pin->pose_in[k] = q[k];
  for (int k = 0; k < 3; ++k) c->pin->pose_in[4 + k] = t[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_out28, c->pin->pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  Pt4* d_out = c->lanes[0].d_full[0];
  LAUNCH(c, KID_KNN_LAST, k_transform_to_end, (in.n + 255) / 256, 256, 0, c->d_query, in.n, c->d_out28, distortion, d_out);
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_out[0], d_out, (size_t)in.n * 16, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

static int run_lm_api(aloam_ctx* c, const double* blocks, int n_blocks, const double x[7], int mode) {
  if (n_blocks < 0 || n_blocks > 2 * kMaxQueries) return ALOAM_ERR_CAPACITY;
  Lane& L = c->lanes[0];
  if (n_blocks > 0) {
    CUDA_CHECK_RET(cudaMemcpyAsync(c->d_packed, blocks, (size_t)n_blocks * 11 * 8, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_PACK_BLOCKS, k_pack_blocks, (n_blocks + 255) / 256, 256, 0, c->d_packed, n_blocks, L.d_blocks);
  }
  for (int k = 0; k < 7; ++k) c->pin->pose_in[k] = x[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_api_pose, c->pin->pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  Batch<LmArgs> b = {};
  b.a[0] = LmArgs{L.d_blocks, nullptr, n_blocks, c->d_api_pose, L.d_summary, c->d_out28, nullptr};
  // blocks from the caller may carry any interpolation ratio; a context emulating a rank (aloam_debug_shard_emulate) with exchange
  // 1 or 2 solves through its exchange, a rank of a real sharded job solves alone
  const int rc = launch_lm_batch(c, false, b, 1, lm_params(c->cfg), mode, 0, true, mode == 0 && c->shard_exchange > 0);
  if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->pose_out, c->d_api_pose, 56, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->ne, c->d_out28, 28 * 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, L.d_summary, sizeof(LmSummary), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

int aloam_normal_equations(aloam_ctx* c, const double* blocks, int n_blocks, const double x[7], double JtJ[36], double Jtr[6],
                           double* cost) {
  if (!c || !x || !JtJ || !Jtr || (n_blocks > 0 && !blocks)) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  int rc = run_lm_api(c, blocks, n_blocks, x, 1);
  if (rc) return rc;
  const double* o = c->pin->ne;
  int k = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) { JtJ[6 * a + b] = o[k]; JtJ[6 * b + a] = o[k]; ++k; }
  for (int a = 0; a < 6; ++a) Jtr[a] = o[21 + a];
  if (cost) *cost = o[27];
  return ALOAM_OK;
}

int aloam_solve(aloam_ctx* c, const double* blocks, int n_blocks, double x[7], double summary7[7], double* trace, int max_trace,
                int* trace_rows) {
  if (!c || !x || (n_blocks > 0 && !blocks)) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  int rc = run_lm_api(c, blocks, n_blocks, x, 0);
  if (rc) return rc;
  for (int k = 0; k < 7; ++k) x[k] = c->pin->pose_out[k];
  const LmSummary& s = c->h_summary[0];
  if (summary7) {
    summary7[0] = s.termination; summary7[1] = s.num_iterations; summary7[2] = s.num_successful; summary7[3] = s.num_jac_evals;
    summary7[4] = 0; summary7[5] = s.initial_cost; summary7[6] = s.final_cost;
  }
  int rows = 0;
  if (trace)
    for (; rows < s.trace_rows && rows < max_trace; ++rows) std::memcpy(trace + (size_t)rows * 8, s.trace[rows], 64);
  if (trace_rows) *trace_rows = rows;
  return ALOAM_OK;
}

// ------------------------------------------------------------------------------------------------ profiling hooks
int aloam_profile_enable(aloam_ctx* c, int on) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  c->prof_on = on != 0;
  c->prof_n = 0;
  for (int k = 0; k < ALOAM_N_KERNEL_IDS; ++k) { c->prof_ms[k] = 0; c->prof_cnt[k] = 0; }
  return ALOAM_OK;
}
int aloam_profile_read(aloam_ctx* c, double* ms_sum, long long* count, const char** names, int capacity) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  int n = capacity < ALOAM_N_KERNEL_IDS ? capacity : ALOAM_N_KERNEL_IDS;
  for (int k = 0; k < n; ++k) { if (ms_sum) ms_sum[k] = c->prof_ms[k]; if (count) count[k] = c->prof_cnt[k]; if (names) names[k] = kKernelNames[k]; }
  return n;
}
long long aloam_launch_count(aloam_ctx* c) { return c ? c->launches : 0; }
// SM-clock cycle counts of the LM solves of the last register / scan_to_pose call: out[5*it] = whole solve, [5*it+1] = evaluation passes, ...
int aloam_debug_lm_cycles(aloam_ctx* c, long long* out, int outer) {
  if (!c || !out) return ALOAM_ERR_INVALID_ARG;
  for (int it = 0; it < outer && it < 4; ++it) { const LmSummary& s = c->h_summary[it]; out[5 * it] = s.cyc_total; out[5 * it + 1] = s.cyc_eval; out[5 * it + 2] = s.cyc_chol; out[5 * it + 3] = s.cyc_plus; out[5 * it + 4] = s.cyc_grad; }
  return ALOAM_OK;
}
// out == NULL arms the time stamps of k_ring_features (they are off by default), otherwise reads them (65 x 8 + 12 values) and disarms
int aloam_debug_feature_cycles(aloam_ctx* c, long long* out64x8) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  cudaSetDevice(c->cfg.device);
  if (!out64x8) { features_debug_enable(1); return ALOAM_OK; }
  features_debug_cycles(out64x8);
  features_debug_enable(0);
  return ALOAM_OK;
}

}  // extern "C"
