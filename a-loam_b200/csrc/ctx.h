// Internal: the context object behind the C ABI and the helpers shared by capi.cu, mapping.cu, cubemap.cu, comm.cu.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <vector>
#include "../../include/aloam_b200.h"
#include "kernels.h"

namespace aloam {
// the buffers of one scan-to-map registration (mapping.cu): the two indexed submaps, the neighbours found by k_map_knn5, the
// residual blocks, the solve summaries and the corner / surf stacks being registered.  The context's set serves the host API
// and lane 0 of the mapper; every other lane of aloam_scan_stream_mapped_batch owns a set of its own.
struct MapReg {
  MapCloud corner, surf;
  float4* nbr;
  BlockRec* blocks;
  LmSummary* summary;   // [4]
  Pt4* stack[2];
};
// one lane of the mapper's index build (the submap clouds) and registration (the stacks' sizes {n_corner, n_surf, total} and
// the pose being refined), all device pointers
struct MapLaneIO {
  MapReg reg;
  const Pt4* sub[2];
  const int* counts3;
  double* pose;
};
// one lane's input to a mapper frame (cubemap.cu): the scan's less-sharp / less-flat clouds and their sizes, its odometry pose
// and the slot of the refined pose, all device pointers; the lane whose cube store the frame runs on, and whether that store
// starts a fresh trajectory with this frame (reset on the device by k_mapper_begin)
struct MapperIn {
  const Pt4* corner;
  const int* nc;
  const Pt4* surf;
  const int* ns;
  const double* odom7;
  double* out7;
  int lane;
  int fresh;
};
}  // namespace aloam

using namespace aloam;

namespace {

constexpr int kMaxSharpPerRing = 12, kMaxLessSharpPerRing = 120, kMaxFlatPerRing = 24;
constexpr int kFusedSharpSlots = 64 * kMaxSharpPerRing;  // 768
constexpr int kFusedFlatSlots = 64 * kMaxFlatPerRing;    // 1536
constexpr int kMaxQueries = ALOAM_MAX_QUERIES;         // API-path capacity for sharp / flat query clouds
constexpr int kProfSlots = 192;                        // kernel launches timed per profile window (one API call)
constexpr int kFeatSlots = 4;                          // feature-set ring of the fused / stream paths
constexpr int kApiLast = kFeatSlots, kApiCur = kFeatSlots + 1;   // feature sets of the per-stage entry points (set_last / extract, register): never the ring's
constexpr int kMaxStreamScans = 4096;                  // scans x lanes per aloam_scan_stream(_batch) call

struct FeatBuf {
  Pt4 *sharp = nullptr, *less_sharp = nullptr, *flat = nullptr, *less_flat = nullptr;
  int* counts = nullptr;           // [4] n_sharp, n_less_sharp, n_flat, n_less_flat (device)
  int *rs_ls = nullptr, *rs_lf = nullptr;  // ring_start tables [65+]
  RabIndex g_ls = {}, g_lf = {};           // (azimuth bucket x ring) indices over less_sharp / less_flat
};

// Everything one trajectory owns on the device.  A context has cfg.max_batch of them; the single-trajectory entry points
// use lane 0, aloam_scan_stream_batch drives lanes 0 .. batch-1 in lockstep with shared launches.
struct Lane {
  float* d_raw[2] = {nullptr, nullptr};          // raw-scan staging, double-buffered by scan parity
  int8_t* d_ring = nullptr;
  int *d_hist = nullptr, *d_offsets = nullptr, *d_scan_start = nullptr, *d_scan_end = nullptr;
  int* d_ring_start[2] = {nullptr, nullptr};
  ScanScalars* d_sc = nullptr;                   // [3]: scan k uses slot k%3 and re-arms the next
  Pt4* d_full[2] = {nullptr, nullptr};           // ring-major cloud, double-buffered for the pipelined stream call
  // per-ring staging sets: in the stream call k_compact(k) runs on the index stream while k_ring_features(k+1) fills the other set
  Pt4 *st_sharp[2] = {}, *st_less_sharp[2] = {}, *st_flat[2] = {}, *st_less_flat[2] = {};
  int* st_counts[2] = {};
  FeatBuf feat[kFeatSlots + 2];                  // [0, kFeatSlots): ring of feature sets (odometry k reads sets k-1 and k while extraction runs ahead) ; kApiLast, kApiCur
  BlockRec* d_blocks = nullptr;
  int* d_corr = nullptr;
  double *d_pose = nullptr, *d_world = nullptr;  // para_q/para_t (laserOdometry.cpp:97-98) and q_w_curr/t_w_curr (:93-94)
  LmSummary* d_summary = nullptr;                // [4]
};

// Pinned scratch of the synchronous entry points: one field per purpose.  The host->device copies from here are
// asynchronous, so two uses that share a field before their synchronise would race.
struct PinnedScratch {
  int feat_counts[4];       // aloam_extract_features: n_sharp, n_less_sharp, n_flat, n_less_flat
  int last_counts[4];       // aloam_odometry_set_last: counts of the "last" feature set
  int ring_err;             // aloam_odometry_set_last: ring-order error word
  int query_counts[4];      // sharp / flat query counts (odometry register / associate)
  GridDyn grid[2];          // aloam_map_upload: corner, surf
  int owned[2];             // sharded map upload: points in owned cells, summed over the ranks
  int shard[3];             // aloam_map_upload_sharded: points kept (corner, surf), error word
  int stack_counts[3];      // scan-to-map stacks: n_corner, n_surf, total
  int mapper_counts[2];     // aloam_mapper_step: input cloud sizes
  int mapper_err;           // aloam_scan_stream_mapped: the mapper's error bits, OR over the call's frames
  int mapper_err_lane[ALOAM_MAX_BATCH];   // aloam_scan_stream_mapped_batch: the same per lane
  int peer_err;             // sharded registration / mapper frames: the peer exchange's error word
  SegDesc vox_seg;          // aloam_voxel_filter: the cloud as the one segment of its filter
  int vox_nseg;             //                     1
  int vox_io[3];            //                     cloud size, filtered size, error word: {n, 0, 0}
  int vox_out_n;            //                     filtered size
  double pose_in[7], pose_out[7];             // pose of the per-stage entry points
  double world[7];                            // fused pipeline: world pose of the scan
  double ne[28];                              // normal equations: J^T J upper 21, J^T r 6, cost
  double mapper_pose_in[7], mapper_pose_out[7];
};

}  // namespace

struct aloam_ctx {
  aloam_config cfg;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int max_points = 0, nblocks_max = 0, max_ring = ALOAM_MAX_RING, n_lanes = 1;
  int sms = 1;                     // SMs of cfg.device (grid-stride launch sizes)
  std::vector<Lane> lanes;
  float* d_curv = nullptr;         // debug outputs of the last extraction (lane 0 only)
  int8_t* d_label = nullptr;
  int* d_scan_nfull = nullptr;     // [kMaxStreamScans] ring-major cloud size of every (scan, lane) of a stream call
  double *d_out28 = nullptr, *d_packed = nullptr;
  double* d_api_pose = nullptr;    // [8] pose of the per-stage entry points (odometry_register, solve, ...): not the warm start of the fused pipeline
  double* d_ident = nullptr;       // [7] identity pose, the source of a lane's odometry reset at a START of the stream driver
  ScanScalars* d_sc_init = nullptr;   // [1] an armed ScanScalars slot (what k_ring_scan arms for the next scan), same use
  int* d_err = nullptr;
  Pt4* d_query = nullptr;
  int* d_knn_idx = nullptr;
  float* d_knn_d = nullptr;
  // multi-GPU sharding of the map (spatial slabs + halo, SURVEY.md 8e): this process's rank / world and its communicator
  int shard_rank = 0, shard_count = 1;
  int shard_exchange = -1;       // >= 0: this context emulates rank shard_rank of shard_count without a communicator (test hook
                                 // aloam_debug_shard_emulate), its LM all-reduce a loopback: 0 k_lm_solve, 1 per evaluation, 2 peer
  void* comm = nullptr;          // ncclComm_t when shard_count > 1 (comm.cu)
  void* peer = nullptr;          // peer-memory exchange of the sharded LM (comm.cu), when enabled
  double* d_lm_tot = nullptr;    // [64] all-reduced normal equations of one evaluation (per-evaluation sharded LM)
  void* d_lm_state = nullptr;    // device-resident trust-region state (per-evaluation sharded LM)
  // map cube store of every lane (cubemap.cu), each created on first use: lane 0 serves the host API and both mapped stream
  // calls, lanes 1 .. max_batch-1 only aloam_scan_stream_mapped_batch
  void* mapper[ALOAM_MAX_BATCH] = {};
  // scan-to-map: the registration set of the host API and mapper lane 0 (uploaded submap with its hash grids, stacks, ...)
  MapReg map = {};
  Pt4* d_map_pts[2] = {nullptr, nullptr};   // staging for maps handed in as host views (device views are indexed in place)
  int max_map = 0, map_slots = 0;
  int map_n[2] = {0, 0};          // points indexed on this rank (corner, surf)
  int map_global_n[2] = {0, 0};   // size of the whole submap (== map_n unless the map is sharded over ranks)
  bool have_map = false;
  bool map_ready = false;         // every buffer of this group is allocated (set last by ensure_map_buffers)
  int* d_stack_counts = nullptr;  // [4] {n_corner, n_surf, total} of the host API's stacks
  double* d_map_pose = nullptr;   // [7] host API: scan-to-map pose being refined (parameters[7], laserMapping.cpp:110)
  double* d_fits = nullptr;       // [queries][14] debug / test records of the line / plane fits
  // aloam_voxel_filter (voxel.cu): a segmented filter of its own (cap = max_points), created on first use
  SegBuffers vox_seg;
  int* d_seg_io = nullptr;        // [3] the segment's size, its filtered size, the filter's error word
  bool vox_seg_ready = false;     // every buffer of this group is allocated
  // pipelined scan stream: ring binning on s_exa, per-ring features on s_ext, compaction + index on s_idx, association + LM
  // on `stream`, host->device copies of the raw scans on s_h2d, scan-to-map on s_map; all chained by events
  cudaStream_t s_ext = nullptr, s_exa = nullptr, s_idx = nullptr, s_h2d = nullptr, s_map = nullptr;
  cudaEvent_t ev_feat[kFeatSlots] = {}, ev_idx[kFeatSlots] = {}, ev_odo[kFeatSlots] = {}, ev_mapdone[kFeatSlots] = {}, ev_h2d[2] = {}, ev_rawfree[2] = {},
              ev_a[2] = {}, ev_b[2] = {}, ev_cmp[2] = {};
  double* h_poses = nullptr;     // pinned [kMaxStreamScans][7]
  double* d_poses = nullptr;     // device [kMaxStreamScans][7]: per-(scan, lane) world poses of a stream call (one D2H at the end)
  double* d_map_poses = nullptr; // device [kMaxStreamScans][7]: map-refined poses (aloam_scan_stream_mapped)
  int* h_scan_nfull = nullptr;   // pinned [kMaxStreamScans]
  // pinned host mirrors
  Pt4* h_out[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  Pt4* h_vox_out = nullptr;     // result of aloam_voxel_filter (never aliases the feature views)
  PinnedScratch* pin = nullptr;
  LmSummary* h_summary = nullptr;   // [n_lanes][4]
  ScanScalars* h_sc = nullptr;      // [n_lanes][3]
  // per-kernel profiler (bench.py roofline leg) + cumulative launch counter
  bool prof_on = false;
  cudaEvent_t prof_ev[2 * kProfSlots] = {};
  int prof_kid[kProfSlots] = {};
  int prof_n = 0;
  double prof_ms[ALOAM_N_KERNEL_IDS] = {};
  long long prof_cnt[ALOAM_N_KERNEL_IDS] = {};
  long long launches = 0;
  // state (all lanes advance in lockstep)
  int parity = 0;         // ScanScalars slot of the next scan
  int frame = 0;          // fused pipeline: scans seen
  int cur = 0;            // fused pipeline: feat[] slot of the most recent scan
  bool have_last = false; // API path: set_last called
  int last_n_full = 0;
  // aloam_scan_stream_lanes: once used, the lockstep calls are refused until aloam_reset_odometry, which clears all of this.
  // A lane runs from its START to the step before its next IDLE; `lane_mapped` is the mode of the call that started it.
  bool lanes_mode = false;
  bool lane_running[ALOAM_MAX_BATCH] = {};
  bool lane_mapped[ALOAM_MAX_BATCH] = {};
  int lockstep_ops[kMaxStreamScans] = {};   // the lane schedule a lockstep stream call hands to the stream driver
  // every resource the context acquires (dalloc, halloc, screate, ecreate, own): aloam_destroy synchronises `streams`, then
  // runs `release` in reverse order of acquisition
  std::vector<cudaStream_t> streams;
  std::vector<std::function<void()>> release;
};

namespace {

enum { KID_CLASSIFY = 0, KID_RING_SCAN, KID_SCATTER, KID_RING_FEATURES, KID_COMPACT, KID_GRID_BUILD, KID_ODOM_ASSOC, KID_LM_SOLVE,
       KID_RING_OFFSETS, KID_KNN_LAST, KID_PACK_BLOCKS, KID_MAP_GRID, KID_MAP_KNN5, KID_VOXEL, KID_MAP_KNN, KID_MAP_FIT, KID_CUBES, KID_LM_SHARD };
const char* const kKernelNames[ALOAM_N_KERNEL_IDS] = {"k_classify", "k_ring_scan", "k_scatter", "k_ring_features", "k_compact",
    "k_rab_build(3 launches)", "k_odom_assoc", "k_lm_solve", "k_ring_offsets", "k_knn_last", "k_pack_blocks", "k_map_grid(4 launches)", "k_map_knn5",
    "k_voxel", "k_map_knn", "k_map_fit", "k_cube_store", "k_lm_shard"};

inline void prof_begin(aloam_ctx* c, int kid) {
  ++c->launches;
  if (c->prof_on && c->prof_n < kProfSlots) { cudaEventRecord(c->prof_ev[2 * c->prof_n], c->stream); c->prof_kid[c->prof_n] = kid; }
}
inline void prof_end(aloam_ctx* c) {
  if (c->prof_on && c->prof_n < kProfSlots) { cudaEventRecord(c->prof_ev[2 * c->prof_n + 1], c->stream); ++c->prof_n; }
}
// call after the stream has been synchronised
inline void prof_collect(aloam_ctx* c) {
  for (int i = 0; i < c->prof_n; ++i) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, c->prof_ev[2 * i], c->prof_ev[2 * i + 1]) == cudaSuccess) { c->prof_ms[c->prof_kid[i]] += ms; ++c->prof_cnt[c->prof_kid[i]]; }
  }
  c->prof_n = 0;
}
#define LAUNCH(c, kid, kernel, grid, block, smem, ...) \
  do { prof_begin(c, kid); kernel<<<grid, block, smem, (c)->stream>>>(__VA_ARGS__); prof_end(c); } while (0)

// launch with an optional programmatic dependency on the previous kernel of the stream (PDL): the grid may become resident
// while its predecessor is still running and blocks in pdl_wait() (common.cuh) until the predecessor has completed and flushed.
template <typename K, typename... Args>
void launch_ex(aloam_ctx* c, int kid, K kernel, dim3 grid, dim3 block, size_t smem, int cluster, bool pdl, Args... args) {
  prof_begin(c, kid);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = c->stream;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (cluster > 1) { at[na].id = cudaLaunchAttributeClusterDimension; at[na].val.clusterDim.x = cluster; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1; ++na; }
  if (pdl && !c->prof_on) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = at; cfg.numAttrs = na;
  cudaLaunchKernelEx(&cfg, kernel, args...);
  prof_end(c);
}

#define LAUNCH_PDL(c, kid, kernel, grid, block, smem, ...) launch_ex(c, kid, kernel, dim3(grid), dim3(block), smem, 1, true, __VA_ARGS__)

// the LM kernel runs as one thread-block cluster per trajectory (distributed-shared-memory reduction, see lm.cu)
constexpr int kLmCluster = 8;

}  // namespace
// Issues one LM solve of trajectories args.a[0 .. lanes-1] on c->stream (comm.cu); every solve of the library goes through here.
// Without `exchange` it is local: k_lm_solve, or k_lm_solve_x when `general` (blocks may carry any interpolation ratio).  With
// `exchange` the normal equations of every evaluation are summed over the ranks of a sharded job (a loopback on a context that
// emulates a rank): one lane in mode 0, through k_lm_solve_x and the peer mailbox when there is one, else per evaluation around
// an all-reduce.  Returns ALOAM_ERR_STATE for an exchange over several lanes and ALOAM_ERR_COMM when the all-reduce fails.
int launch_lm_batch(aloam_ctx* c, bool pdl, const aloam::Batch<aloam::LmArgs>& args, int lanes, const aloam::LmParams& lp, int mode, int integrate,
                    bool general, bool exchange);
// the error word of the peer exchange (a peer that did not answer in time), on c->stream: cleared at the start of every call
// that registers against a sharded map, copied to pinned *dst with its pose (*dst = 0 without the peer exchange)
int peer_err_reset(aloam_ctx* c);
int peer_err_fetch(aloam_ctx* c, int* dst);
void vox_seg_filter(aloam_ctx* c, int nb, const aloam::SegFilter* f, aloam::SegBuffers* const* b, int S_upper, int n_upper, int per_seg_upper);
int vox_seg_alloc(aloam_ctx* c, aloam::SegBuffers& b, size_t cap);
int mapper_step_device(aloam_ctx* c, int nb, const MapperIn* in, int n_upper_c, int n_upper_s);
int mapper_ensure_lanes(aloam_ctx* c, int nb);
int* mapper_err_acc(aloam_ctx* c, int lane);
int ensure_map_buffers(aloam_ctx* c);
int map_reg_alloc(aloam_ctx* c, MapReg* r);
void map_index_build(aloam_ctx* c, int nb, const MapLaneIO* io, int n_upper);
int map_shard_index_device(aloam_ctx* c, Pt4* const sub[2], const int* n_sub, int n_upper, int* err_word);
int map_register_device(aloam_ctx* c, int nb, const MapLaneIO* io, int nq_upper);
namespace {

// a rank of a sharded job: joined to a world of several ranks by a communicator, or emulating a rank (aloam_debug_shard_emulate)
inline bool sharded_job(const aloam_ctx* c) { return c->shard_count > 1 || c->shard_exchange >= 0; }
// the scan-to-map LM exchanges its normal equations: on a rank of a sharded job, and on a context that emulates a rank with
// exchange 1 or 2
inline bool sharded_lm(const aloam_ctx* c) { return c->shard_exchange < 0 ? c->shard_count > 1 : c->shard_exchange > 0; }

LmParams lm_params(const aloam_config& c) {
  LmParams p;
  p.max_iters = c.inner_iters; p.huber_a = c.huber;
  p.initial_radius = 1e4; p.max_radius = 1e16; p.min_radius = 1e-32;
  p.min_relative_decrease = 1e-3; p.min_lm_diagonal = 1e-6; p.max_lm_diagonal = 1e32;
  p.function_tolerance = 1e-6; p.gradient_tolerance = 1e-10; p.parameter_tolerance = 1e-8;
  p.max_invalid = 5;
  return p;
}

// acquisition helpers: what they return belongs to the context and is released by aloam_destroy
inline void own(aloam_ctx* c, std::function<void()> f) { c->release.push_back(std::move(f)); }
template <typename T> cudaError_t dalloc(aloam_ctx* c, T** p, size_t n) {
  const cudaError_t e = cudaMalloc((void**)p, n * sizeof(T));
  if (e == cudaSuccess) { void* q = *p; own(c, [q] { cudaFree(q); }); }
  return e;
}
template <typename T> cudaError_t halloc(aloam_ctx* c, T** p, size_t n) {
  const cudaError_t e = cudaMallocHost((void**)p, n * sizeof(T));
  if (e == cudaSuccess) { void* q = *p; own(c, [q] { cudaFreeHost(q); }); }
  return e;
}
inline cudaError_t screate(aloam_ctx* c, cudaStream_t* s) {
  const cudaError_t e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
  if (e == cudaSuccess) { const cudaStream_t q = *s; c->streams.push_back(q); own(c, [q] { cudaStreamDestroy(q); }); }
  return e;
}
inline cudaError_t ecreate(aloam_ctx* c, cudaEvent_t* ev, unsigned flags) {
  const cudaError_t e = cudaEventCreateWithFlags(ev, flags);
  if (e == cudaSuccess) { const cudaEvent_t q = *ev; own(c, [q] { cudaEventDestroy(q); }); }
  return e;
}

int upload_cloud(aloam_ctx* c, aloam_cloud_view v, Pt4* dst, int capacity) {
  if (v.n < 0 || (v.n > 0 && !v.data) || (v.stride_floats != 4 && v.stride_floats != 8 && v.n > 0)) return ALOAM_ERR_INVALID_ARG;
  if (v.n > capacity) return ALOAM_ERR_CAPACITY;
  if (v.n == 0) return ALOAM_OK;
  if (v.stride_floats == 4) {
    CUDA_CHECK_RET(cudaMemcpyAsync(dst, v.data, (size_t)v.n * 16, cudaMemcpyDefault, c->stream));   // host or device source
  } else {
    CUDA_CHECK_RET(cudaMemcpy2DAsync(dst, 16, v.data, (size_t)v.stride_floats * 4, 16, v.n, cudaMemcpyDefault, c->stream));
  }
  return ALOAM_OK;
}

LastCloud last_corner(const FeatBuf& f) { return LastCloud{f.less_sharp, f.counts + 1, f.g_ls}; }
LastCloud last_surf(const FeatBuf& f) { return LastCloud{f.less_flat, f.counts + 3, f.g_lf}; }

void fill_stats_from(const LmSummary* h_summary, aloam_stats* st, int outer, int flags, float ms) {
  if (!st) return;
  std::memset(st, 0, sizeof(*st));
  st->flags = flags;
  st->ms_total = ms;
  for (int it = 0; it < outer && it < 4; ++it) {
    const LmSummary& s = h_summary[it];
    st->lm_iters += s.num_iterations;
    st->accepted_steps += s.num_successful;
    st->termination[it] = s.termination;
    if (it == outer - 1) {
      st->n_corner_corr = s.n_edge; st->n_plane_corr = s.n_plane;
      st->init_cost = s.initial_cost; st->final_cost = s.final_cost;
      if (s.n_edge + s.n_plane < 10) st->flags |= ALOAM_FLAG_FEW_CORRESPONDENCES;
    }
  }
}
inline void fill_stats(aloam_ctx* c, aloam_stats* st, int outer, int flags, float ms) { fill_stats_from(c->h_summary, st, outer, flags, ms); }

int check_view(const aloam_cloud_view& v) {
  if (v.n < 0) return ALOAM_ERR_INVALID_ARG;
  if (v.n > 0 && (!v.data || (v.stride_floats != 4 && v.stride_floats != 8))) return ALOAM_ERR_INVALID_ARG;
  return ALOAM_OK;
}

}  // namespace
