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
#include "snapshot.h"

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
  int localise;   // the lane registers against the context's prior map: its frame state is its locator's, not a cube store's
  int seed;       // the lane starts a mapping trajectory with this frame on a copy of the prior map, from T_wmap_wodom Lane::init
                  // (aloam_lane_map_on_prior): its store is seeded before the frame, `fresh` is off
};
// what the registration of localising lanes searches instead of each lane's indexed submap: the prior map's grids, and per
// lane the window tables and centre cube k_locate_begin left in its frame state
struct PriorSearch {
  PriorGrid grid;
  const int* win[ALOAM_MAX_BATCH][2];
  const int* ctr[ALOAM_MAX_BATCH];
};
// the head of an LmSummary, termination through final_cost: what a frame's stats are made of
struct LmHead {
  int termination, num_iterations, num_successful, num_jac_evals;
  int n_edge, n_plane;
  double initial_cost, final_cost;
};
// one row of a mapped stream call as k_map_rows (cubemap.cu) and the tracking score (rows.cu, k_inlier_score in reloc.cu) leave it
// on the device: the frame's flags and error word, its window and stack sizes, the summaries of its outer iterations and its
// prior-map inlier score (-1: not scored; k_inlier_score adds to 0).  With recovery on (aloam_set_recovery), a localising row also
// holds what its recovery did: k_recover_cand (recover.cu) sets rec_triggered, k_recover_adopt (cubemap.cu) the rest of a
// triggered row.
struct MapRowRec {
  int flags, err, n_valid, n_sub[2], n_stack[2], score, n_score, pad;
  LmHead lm[4];
  int rec_triggered, rec_best, rec_best_score, rec_adopted;
  double rec_pose[7];
};
// one hypothesis set of k_reloc_score / k_reloc_topk (reloc.cu): n_hyp normalised poses (7 doubles each) scored against the
// stacks (sizes counts[0], counts[1]) into score[h] through warp_inliers (grid.cuh), as inlier_score_device scores one pose;
// part (may be null): the CTAs' best keys, kRelocTop per CTA; best: the best keys of the set; gate (may be null): the set is
// ranked only when *gate != 0 -- its CTAs leave at once otherwise
struct RelocRec {
  const double* hyp;
  int n_hyp;
  const Pt4* stack[2];
  const int* counts;
  int* score;
  unsigned long long* part;
  unsigned long long* best;
  const int* gate;
};
// one record of k_inlier_score (reloc.cu): stacks of sizes counts[0], counts[1] scored at one pose against the corner and surf
// grids; the count is added to *score
struct ScoreRec {
  const Pt4* stack[2];
  const int* counts;
  const double* pose;
  GridTable grid[2];
  int* score;
};
// Buffers that a later call replaces as a whole (a larger table, a new map): a replacement group is filled on the side and
// swapped in only when every allocation in it succeeded; the group it replaces is freed as a whole by its destructor.  Nothing
// here synchronises: an owner drains the work that reads a group's buffers before it frees them.
class BufGroup {
 public:
  BufGroup() = default;
  BufGroup(BufGroup&& o) noexcept { swap(o); }
  BufGroup& operator=(BufGroup&& o) noexcept { BufGroup t(std::move(o)); swap(t); return *this; }
  ~BufGroup() {
    for (void* p : dev_) cudaFree(p);
    for (void* p : pinned_) cudaFreeHost(p);
  }
  // n elements of T in device / page-locked host memory, recorded in the group; false (the error cleared, *p null) on failure
  template <typename T> bool dev(T** p, size_t n) { return keep(cudaMalloc((void**)p, n * sizeof(T)), (void**)p, dev_); }
  template <typename T> bool pinned(T** p, size_t n) { return keep(cudaMallocHost((void**)p, n * sizeof(T)), (void**)p, pinned_); }
  void swap(BufGroup& o) noexcept { dev_.swap(o.dev_); pinned_.swap(o.pinned_); }
  bool empty() const { return dev_.empty() && pinned_.empty(); }

 private:
  static bool keep(cudaError_t e, void** p, std::vector<void*>& list) {
    if (e != cudaSuccess) { cudaGetLastError(); *p = nullptr; return false; }
    list.push_back(*p);
    return true;
  }
  std::vector<void*> dev_, pinned_;
};
struct ExportLayout;   // cubemap.cu: where the segments of a store export are in the export and in the store
struct LaneFrame;      // cubemap.cu: what a scan-to-map frame runs on -- frame state, registration set, stack filter
struct Mapper;         // cubemap.cu: a lane's cube store, one frame and the store's buffers
struct PriorMap;       // cubemap.cu: the context's prior map, frozen and indexed
struct Relocaliser;    // reloc.cu: the scratch of aloam_prior_relocalise
struct Recovery;       // recover.cu: the setting and buffers of aloam_set_recovery
struct Place;          // place.cu: the keyframe tables, database and scratch of place recognition (aloam_set_place)
struct Loop;           // loop.cu: the setting, keyframe clouds and registration sets of loop verification (aloam_set_loops)
}  // namespace aloam

using namespace aloam;

namespace {

// per-ring caps of the feature clouds; a context's query slots and staging sets are ring_w (64 or 128) times these
constexpr int kMaxSharpPerRing = 12, kMaxLessSharpPerRing = 120, kMaxFlatPerRing = 24;
constexpr int kMaxQueries = ALOAM_MAX_QUERIES;         // API-path capacity for sharp / flat query clouds
constexpr int kProfSlots = 192;                        // kernel launches timed per profile window (one API call)
constexpr int kFeatSlots = 4;                          // feature-set ring of the fused / stream paths
constexpr int kApiLast = kFeatSlots, kApiCur = kFeatSlots + 1;   // feature sets of the per-stage entry points (set_last / extract, register): never the ring's
constexpr int kMaxStreamScans = 4096;                  // scans x lanes per aloam_scan_stream(_batch) call
constexpr int kRelocTop = ALOAM_MAX_BATCH;             // best keys k_reloc_score keeps per CTA and k_reloc_topk returns

struct FeatBuf {
  Pt4 *sharp = nullptr, *less_sharp = nullptr, *flat = nullptr, *less_flat = nullptr;
  int* counts = nullptr;           // [4] n_sharp, n_less_sharp, n_flat, n_less_flat (device)
  RabIndex g_ls = {}, g_lf = {};           // (azimuth bucket x ring) indices over less_sharp / less_flat
  Pt4* full = nullptr;             // ring-major cloud of a mapped scan, kept for its registered cloud (created by aloam_set_registered_sink)
};

// Row k * nb + l of a stream call: scan k of lane l, as the call will run it
struct StreamRow {
  int op;               // ALOAM_LANE_*
  int scan;             // index of the scan in its trajectory (-1: an IDLE row)
  bool mapped;          // a mapped call's scan that goes to the mapper (or its lane's locator); the others get a high-frequency pose
  bool localise;        // a mapped call's scan that registers against the prior map
  bool seed;            // a mapped call's START that maps on a copy of the prior map (consumes an aloam_lane_map_on_prior arming)
  long long reg_begin;  // where the row's registered cloud begins in the sink: the sum of raws[r'].n over the mapped rows r' before it
};
// the rows of a stream call, built before anything is issued (room for all n in one allocation); reg_total: the points of every
// mapped row's registered cloud
struct StreamTable { std::vector<StreamRow> rows; long long reg_total = 0; explicit StreamTable(size_t n = 0) { rows.reserve(n); } };
// the ALOAM_ROW_* of a row (aloam_map_row::kind)
inline int row_kind(const StreamRow& r) { return r.op == ALOAM_LANE_IDLE ? ALOAM_ROW_IDLE : !r.mapped ? ALOAM_ROW_SKIPPED : r.localise ? ALOAM_ROW_LOCALISED : ALOAM_ROW_MAPPED; }
// The last mapped stream call, all its readers read: scan_stream_run takes over its rows and clears the flags before it issues
// anything, sets them once the call has drained; a mapped lanes call refused with a scan that cannot run clears `records`.
struct MappedCall {
  StreamTable table; int n_scans = 0, nb = 0;   // n_scans x nb rows
  std::vector<int> reg_count;    // per row: points of its registered cloud in the sink (0 without a sink or for a row not mapped)
  bool registered = false;       // aloam_registered_rows may read the table and reg_count
  bool records = false;          // aloam_map_rows and aloam_recovery_rows may read the table and the pinned row table h_rows
  bool recovered = false;        // the call ran recovery (aloam_set_recovery)
  bool places = false;           // aloam_place_rows may read the table and the pinned place rows (the call recorded keyframes)
  bool loops = false;            // aloam_loop_rows may read the table and the pinned loop rows (the call verified loops)
  // a reader's check: ALOAM_ERR_STATE while its flag is off, ALOAM_ERR_INVALID_ARG for a row count other than the call's
  int check(bool readable, int rows) const { return !readable ? ALOAM_ERR_STATE : rows != n_scans * nb ? ALOAM_ERR_INVALID_ARG : ALOAM_OK; }
};

// Where a lane is in the schedule of the stream calls.  A lane of aloam_scan_stream_lanes runs from its START to the step before
// its next IDLE; `mapped` is the mode of the call that started it; `localising`: the trajectory it runs (or ran last) registers
// against the prior map, fixed at its START; `arm`: what its next mapped START does with Lane::init -- localise from it
// (aloam_lane_localise) or map on a copy of the prior map from it (aloam_lane_map_on_prior); the later arming replaces the other.
// `scan`: index of its next scan in its trajectory (0 at a START), which every stream call advances; scan j goes to the mapper
// when j % cfg.mapping_skip_frame == 0.  aloam_reset_odometry puts back the default.
enum LaneArm { ARM_NONE = 0, ARM_LOCALISE, ARM_MAP_ON_PRIOR };
struct LaneSched {
  bool running = false, mapped = false, localising = false;
  int arm = ARM_NONE;
  int scan = 0;
};

// Everything one trajectory owns.  A context has cfg.max_batch of them; the single-trajectory entry points use lane 0,
// aloam_scan_stream_batch drives lanes 0 .. batch-1 in lockstep with shared launches.
struct Lane {
  LaneSched sched;
  // its cube store and its locator, the frame its localising trajectories run on (cubemap.cu), each created on first use: lane
  // 0's store serves the host API and both mapped stream calls; a lane that only localises has no store
  Mapper* mapper = nullptr;
  LaneFrame* locator = nullptr;
  double init[7] = {};   // the T_wmap_wodom an armed START starts from (aloam_lane_localise, aloam_lane_map_on_prior)
  // the locator holds the window of a localising frame against the current prior map (aloam_debug_prior_associate); set by the
  // frame, cleared when the prior map is released
  bool window = false;
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
  int locate_err_lane[ALOAM_MAX_BATCH];   // aloam_scan_stream_lanes: the same of every lane's localising frames
  int peer_err;             // sharded registration / mapper frames: the peer exchange's error word
  SegDesc vox_seg;          // aloam_voxel_filter: the cloud as the one segment of its filter
  int vox_nseg;             //                     1
  int vox_io[3];            //                     cloud size, filtered size, error word: {n, 0, 0}
  int vox_out_n;            //                     filtered size
  long long export_total;   // aloam_mapper_export: points of the export
  double pose_in[7], pose_out[7];             // pose of the per-stage entry points
  double world[7];                            // fused pipeline: world pose of the scan
  double ne[28];                              // normal equations: J^T J upper 21, J^T r 6, cost
  double mapper_pose_in[7], mapper_pose_out[7];
  SnapHeader snap;          // aloam_lane_save / _restore: the snapshot's header
  int snap_counts[4];       //                             counts of the lane's "last" feature set
  SnapLocalise snap_loc;    // aloam_lane_save_localising / _restore: the locator section of a format-2 snapshot
};

}  // namespace

struct aloam_ctx {
  aloam_config cfg;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int max_points = 0, nblocks_max = 0, max_ring = ALOAM_MAX_RING, n_lanes = 1;
  // ring width (kernels.h ring_width): 64, or 128 for a context of aloam_create_wide with more than 64 rings.  The fused paths'
  // query slots (sharp 12 / flat 24 per ring: 768 / 1536 at 64) and the less-sharp bound (120 per ring) follow from it.
  int ring_w = 64;
  int fused_sharp_slots() const { return ring_w * kMaxSharpPerRing; }
  int fused_flat_slots() const { return ring_w * kMaxFlatPerRing; }
  int less_sharp_upper() const { return ring_w * kMaxLessSharpPerRing; }
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
  // aloam_voxel_filter (voxel.cu): a segmented filter of its own (cap = max_points), created on first use, published complete
  SegBuffers vox_seg;
  int* d_seg_io = nullptr;        // [3] the segment's size, its filtered size, the filter's error word
  // pipelined scan stream: ring binning on s_exa, per-ring features on s_ext, compaction + index on s_idx, association + LM
  // on `stream`, host->device copies of the raw scans on s_h2d, scan-to-map on s_map; all chained by events
  cudaStream_t s_ext = nullptr, s_exa = nullptr, s_idx = nullptr, s_h2d = nullptr, s_map = nullptr;
  // ev_mapdone[s]: the last mapper frame that read feature slot s (recorded only by steps that map a lane); ev_mapend: everything
  // a call issued on s_map, high-frequency poses included
  cudaEvent_t ev_feat[kFeatSlots] = {}, ev_idx[kFeatSlots] = {}, ev_odo[kFeatSlots] = {}, ev_mapdone[kFeatSlots] = {}, ev_h2d[2] = {}, ev_rawfree[2] = {},
              ev_a[2] = {}, ev_b[2] = {}, ev_cmp[2] = {}, ev_mapend = nullptr;
  // registered full-resolution clouds of the mapped streams (aloam_set_registered_sink): the sink (device or page-locked host memory,
  // written through its device address) and its capacity in points; ev_stash[b]: the copy of ring-major cloud b into the feature
  // slot's stash is done (created with the stash).  The rows' places in the sink are in last_mapped.
  Pt4* reg_sink = nullptr;
  long long reg_cap = 0;
  cudaEvent_t ev_stash[2] = {};
  // per-row records of the mapped stream calls (aloam_set_map_rows, rows.cu): the setting, and the device row table and its pinned
  // copy ([kMaxStreamScans] each, created by the first call that turns recording on)
  bool rows_on = false;
  float rows_inlier_sq = 1.f;
  int rows_max_score = 0;
  MapRowRec* d_rows = nullptr;
  MapRowRec* h_rows = nullptr;
  // recovery of localising lanes (aloam_set_recovery, recover.cu): on only while rows are scored; its buffers, created on first use
  bool rec_on = false;
  Recovery* recover = nullptr;
  // place recognition (aloam_set_place, place.cu): keyframes recorded by the mapped stream calls while place_on; the tables,
  // database and scratch, created on first use
  bool place_on = false;
  Place* place = nullptr;
  // loop verification (aloam_set_loops, loop.cu): keyframe clouds and in-stream verification while loop_on (only with place_on);
  // its buffers, created by the call that turns it on
  bool loop_on = false;
  Loop* loop = nullptr;
  MappedCall last_mapped;   // the rows of the last mapped stream call and which of its readers may read them
  // exports of a lane's store (aloam_mapper_export, lane snapshots): the layout of the last one and the staging buffer of host
  // memory, created on first use
  ExportLayout* d_export_layout = nullptr;
  Pt4* d_export_stage = nullptr;
  double* h_poses = nullptr;     // pinned [kMaxStreamScans][7]
  double* d_poses = nullptr;     // device [kMaxStreamScans][7]: per-(scan, lane) world poses of a stream call (one D2H at the end)
  double* d_map_poses = nullptr; // device [kMaxStreamScans][7]: map-refined poses (aloam_scan_stream_mapped)
  int* h_scan_nfull = nullptr;   // pinned [kMaxStreamScans]
  // pinned host mirrors
  Pt4* h_out[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  Pt4* h_vox_out = nullptr;     // result of aloam_voxel_filter (never aliases the feature views)
  Pt4* h_cube = nullptr;        // aloam_mapper_debug_cube of a cube beyond max_points (cube growth), created on first use
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
  bool have_last = false; // API path: set_last called
  int last_n_full = 0;
  // aloam_scan_stream_lanes: once used, the lockstep calls are refused until aloam_reset_odometry, which clears it and every
  // lane's schedule state
  bool lanes_mode = false;
  // the stack filters of mapping and localising frames run on s_stack, forked from and joined to the frame's stream by these
  // events (cubemap.cu; created with the first cube store or locator)
  cudaStream_t s_stack = nullptr;
  cudaEvent_t ev_stack_fork = nullptr, ev_stack_join = nullptr;
  // localisation (cubemap.cu): the context's prior map, released by prior_map_release
  PriorMap* prior = nullptr;
  bool prior_owned = false;       // prior_map_release is on the release list
  Relocaliser* reloc = nullptr;   // aloam_prior_relocalise (reloc.cu), created on first use, released through `release`
  // every resource the context acquires (dalloc, halloc, screate, ecreate, own): aloam_destroy synchronises `streams`, then
  // runs `release` in reverse order of acquisition
  std::vector<cudaStream_t> streams;
  std::vector<std::function<void()>> release;
  // aloam_lane_save / _restore of mapped lanes: the store table of a snapshot, pinned and on the device, created on first use
  SnapStore* h_snap_store = nullptr;
  SnapStore* d_snap_store = nullptr;
  // the seeded STARTs of a step (aloam_lane_map_on_prior): the ALOAM_EXPORT_MAP layout of record l's new store, [n_lanes], created
  // by the first stream call that seeds a store
  ExportLayout* d_seed_layout = nullptr;
  // aloam_set_cube_growth: what a lane's store takes at its next mapped START (lane 0 of the host API at aloam_mapper_reset)
  bool cube_growth = false;
};

namespace {

enum { KID_CLASSIFY = 0, KID_RING_SCAN, KID_SCATTER, KID_RING_FEATURES, KID_COMPACT, KID_GRID_BUILD, KID_ODOM_ASSOC, KID_LM_SOLVE,
       KID_RING_OFFSETS, KID_KNN_LAST, KID_PACK_BLOCKS, KID_MAP_GRID, KID_MAP_KNN5, KID_VOXEL, KID_MAP_KNN, KID_MAP_FIT, KID_CUBES, KID_LM_SHARD, KID_MAP_KNN5_PRIOR,
       KID_PRIOR_BUILD, KID_RELOC, KID_RELOC_TOPK, KID_MAP_ROWS, KID_TRACK_SCORE, KID_RECOVER_CAND, KID_RECOVER_ADOPT,
       KID_PRIOR_DIGEST, KID_PLACE_GATE, KID_PLACE_DIST, KID_PLACE_BEST, KID_LOOP_KEEP, KID_LOOP_VERIFY };
const char* const kKernelNames[ALOAM_N_KERNEL_IDS] = {"k_classify", "k_ring_scan", "k_scatter", "k_ring_features", "k_compact",
    "k_rab_build(3 launches)", "k_odom_assoc", "k_lm_solve", "k_ring_offsets", "k_knn_last", "k_pack_blocks", "k_map_grid(4 launches)", "k_map_knn5",
    "k_voxel", "k_map_knn", "k_map_fit", "k_cube_store", "k_lm_shard", "k_map_knn5_prior",
    "k_prior_build", "k_reloc_score", "k_reloc_topk", "k_map_rows", "k_track_score", "k_recover_cand", "k_recover_adopt",
    "k_prior_digest", "k_place_gate(describe)", "k_place_dist", "k_place_best", "k_loop_keep", "k_loop_gather/score/finish"};

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
int vox_seg_alloc(aloam_ctx* c, BufGroup& g, aloam::SegBuffers& b, size_t cap);
// voxel.cu: the segmented filter's stable radix sort over one key array of up to n_upper keys (the prior-map build), and the ints
// of histogram it needs for n keys
int vox_radix_sort(aloam_ctx* c, int kid, unsigned* k0, int* v0, unsigned* k1, int* v1, const int* n_dev, int n_upper, int bits, int* hist);
size_t vox_radix_hist_ints(int n);
int mapper_step_device(aloam_ctx* c, int nb, const MapperIn* in, int n_upper_c, int n_upper_s);
int mapper_high_freq_device(aloam_ctx* c, int nb, const MapperIn* in);
int mapper_register_full_device(aloam_ctx* c, int nb, const MapperIn* in, const Pt4* const* src, const int* const* n_full, Pt4* const* dst, int n_upper);
// per-row records (aloam_set_map_rows): the rows of the nb records of the frame just issued (cubemap.cu), and the prior-map inlier
// score of its localising records at their map poses (rows.cu; n_upper_c / n_upper_s bound the stacks as for the frame)
int map_rows_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, int max_score);
int track_score_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, int n_upper_c, int n_upper_s);
// relocalisation scoring (reloc.cu), one hypothesis set per record in blockIdx.z: k_reloc_score over nrec sets with `ctas` CTAs
// each (max_pts scoring points per type, inliers at float d2 < inlier_sq); k_reloc_topk: the `rounds` best keys of each set's
// ctas x kRelocTop CTA keys.  reloc_score_ctas: the CTAs a set of n_hyp hypotheses is scored with (at most one resident wave).
void reloc_score_device(aloam_ctx* c, int nrec, const Batch<RelocRec>& B, int ctas, int max_pts, float inlier_sq);
void reloc_topk_device(aloam_ctx* c, int nrec, const Batch<RelocRec>& B, int ctas, int rounds);
int reloc_score_ctas(aloam_ctx* c, int n_hyp);
// one pose per record (reloc.cu): k_inlier_score under profile id kid over records B.a[0 .. nb-1], parallel over the scoring
// points (max_pts per type; m_upper: the host's bound on any record's scoring points sizes the grid), inliers at float d2 <
// inlier_sq added to each record's *score; tracking scores (rows.cu) and loop verification (loop.cu) launch it
void inlier_score_device(aloam_ctx* c, int kid, int nb, const Batch<ScoreRec>& B, long long m_upper, int max_pts, float inlier_sq);
// recovery of localising lanes (recover.cu): after track_score_device, the recovery of the frame's nb localising records, whose
// scored rows are rows[l]; and its last kernel (cubemap.cu), which adopts record l's best candidate (of cand[l], best key *best[l])
int recover_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows);
int recover_adopt_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, const double* const* cand,
                         const unsigned long long* const* best, float accept_frac);
// place recognition (place.cu): after the mapping frame of nb records just issued, the keyframe gate, descriptor and loop query of
// each (scan[l]: its scan index, start[l]: it STARTs a trajectory, which clears its lane's table first; rows[l]: its place row);
// and the clearing of lane `lane`'s table (-1: every lane), on c->stream
// (*n_upper, when not null: the host bound on the keyframes any record's loop query searches; <= 0 when no record can have one)
int place_record_device(aloam_ctx* c, int nb, const MapperIn* in, const int* scan, const bool* start, aloam_place_row* const* rows,
                        int* n_upper = nullptr);
int place_clear(aloam_ctx* c, int lane);
aloam_place_row* place_rows_device(aloam_ctx* c);
aloam_place_row* place_rows_host(aloam_ctx* c);
// lane `lane`'s keyframe table (place recording has been on): its records and count on the device, the keyframes it takes and the
// loop query's exclude_recent
struct PlaceTable { const char* rec; const int* count; int cap; int exclude; };
PlaceTable place_table(aloam_ctx* c, int lane);
// loop verification (loop.cu): after place_record_device of the mapping frame of nb records, the keyframe clouds of its keyframe
// rows and the verification of its triggered rows (prow[l]: record l's place row; n_upper: the bound place_record_device returned),
// on c->stream; the clearing of lane `lane`'s clouds goes with its place table (nothing to do on the device)
int loop_record_device(aloam_ctx* c, int nb, const MapperIn* in, const aloam_place_row* const* prow, size_t r0, int n_upper);
void* loop_rows_device(aloam_ctx* c);
void* loop_rows_host(aloam_ctx* c);
size_t loop_row_bytes();
// which lanes' candidate scores belong to a triggered row of the last mapped stream call (recover.cu; none while its records
// cannot be read or it ran no recovery)
void recover_call_done(aloam_ctx* c);
// the cube store of lane `lane`, created on first use with the state of a fresh trajectory (a failure publishes nothing)
int mapper_ensure(aloam_ctx* c, int lane);
// the layouts of seeded STARTs (aloam_ctx::d_seed_layout), created on first use
int mapper_seed_ensure(aloam_ctx* c);
// the frame lane `lane` runs on in mode `localise`: its locator, else its cube store's frame; null when the lane has none
LaneFrame* lane_frame(const aloam_ctx* c, int lane, bool localise);
// what frame f's latest run left on the device: its filtered corner / surf stacks (sensor frame), their sizes (counts[0],
// counts[1]), its flags followed by its error word (2 ints) and its solve summaries; and the OR of its error words over one
// mapped stream call
struct FrameView { const Pt4* stack[2]; const int* counts; const int* flags; const LmSummary* summary; int* err_acc; };
FrameView frame_view(const LaneFrame* f);
// localisation against the prior map (cubemap.cu): a new locator; a lane's locator, created on first use; one frame of nb
// localising records on the current stream, record l on locator loc[l] (in[l].fresh: it starts a trajectory with this frame,
// from T_wmap_wodom init[l])
int locator_create(aloam_ctx* c, LaneFrame** out);
int locator_ensure(aloam_ctx* c, int lane);
int locate_step_device(aloam_ctx* c, int nb, const MapperIn* in, LaneFrame* const* loc, const double* const* init, int n_upper_c, int n_upper_s);
// the stack filters of a localising frame alone, for locator f on the clouds of `in`, joined to the current stream: the
// filtered stacks and their sizes as frame_view reports them (a stack filter's error bit joins the locator's next frame)
int locator_stacks_device(aloam_ctx* c, LaneFrame* f, const MapperIn& in, int n_upper_c, int n_upper_s);
// the hash grids of the context's prior map (it exists)
PriorGrid prior_grid(const aloam_ctx* c);
// the checks and normalisation of an initial T_wmap_wodom (aloam_lane_localise, aloam_prior_relocalise): false for a non-finite
// value or a zero quaternion, else out = (q / |q|, t), |q|^2 summed in index order
inline bool map_pose_normalise(const double q[4], const double t[3], double out[7]) {
  double n2 = 0;
  for (int k = 0; k < 4; ++k) { if (!std::isfinite(q[k])) return false; n2 += q[k] * q[k]; }
  for (int k = 0; k < 3; ++k) if (!std::isfinite(t[k])) return false;
  if (!(n2 > 0) || !std::isfinite(n2)) return false;
  const double n = std::sqrt(n2);
  for (int k = 0; k < 4; ++k) out[k] = q[k] / n;
  for (int k = 0; k < 3; ++k) out[4 + k] = t[k];
  return true;
}
// the search of lane `lane`'s latest localising frame as record 0 of *ps: the prior map's grids, the window tables and centre cube
// in the lane's locator.  ALOAM_ERR_STATE without a prior map or when the lane has run no localising frame against it.
int locator_prior_search(aloam_ctx* c, int lane, PriorSearch* ps);
inline bool any_lane_localising(const aloam_ctx* c) {
  for (const Lane& L : c->lanes) if (L.sched.running && L.sched.localising) return true;
  return false;
}
// snapshot.cu: the kind of a caller's snapshot buffer (1 device memory of the context's device, 0 host memory, -1 unusable), and
// the host checks of aloam_lane_restore on the snapshot at b -- header (left in c->pin->snap), configuration against the
// context's and, mapped, the store table (left in c->h_snap_store); need_mapped: an unmapped snapshot is refused too.
// *store = byte offset of the store section.
int snapshot_buffer_kind(const aloam_ctx* c, const void* p);
int snapshot_validate(aloam_ctx* c, const char* b, long long n_bytes, int kind, bool need_mapped, long long* store);
// snapshot.cu: the map position p (T_wmap_wodom times a world pose) may start a mapping frame of a store with centre offsets cen --
// its centre cube lies at most kCubeSlack cubes outside the buffer on every axis, so the frame's shift loop ends
bool map_position_fits(const double p[3], const int cen[3]);
void mapper_slab_caps(const aloam_ctx* c, int cap[2]);
// cubemap.cu: the largest run of a lane store per type (2^ord[t] slabs) under cube growth `growth`
void mapper_run_orders(const aloam_ctx* c, bool growth, int ord[2]);
int mapper_store_tables(aloam_ctx* c, int lane, SnapStore* head, int* growth);
int mapper_store_points(aloam_ctx* c, int lane, long long n, char* dst, bool device);
int mapper_store_restore(aloam_ctx* c, int lane, const SnapStore* head, const char* pts, bool device, bool growth);
// cubemap.cu: what names the context's prior map in a localising snapshot -- its centre offsets, its points per type and its
// digest (aloam_prior_map_digest: computed on the first call, then kept with the map).  ALOAM_ERR_STATE without a prior map.
int prior_map_identity(aloam_ctx* c, int cen[3], long long n[2], unsigned long long* digest);
// cubemap.cu: the T_wmap_wodom of lane `lane`'s locator (it exists) into dst[7] (host memory: q xyzw, t), on c->stream, not
// synchronised; and the locator's frame state set to what a fresh localising START leaves before its first frame, with
// T_wmap_wodom = T[7] and the prior map's centre offsets (it exists), on c->stream
int locator_map_pose(aloam_ctx* c, int lane, double* dst);
int locator_restore(aloam_ctx* c, int lane, const double T[7]);
int index_last_clouds(aloam_ctx* c, int lane, int slot, int n_ls, int n_lf);
int ensure_map_buffers(aloam_ctx* c);
int map_reg_alloc(BufGroup& g, MapReg* r, size_t queries, size_t bound, unsigned slots);
void map_index_build(aloam_ctx* c, int nb, const MapLaneIO* io, int n_upper);
int map_shard_index_device(aloam_ctx* c, Pt4* const sub[2], const int* n_sub, int n_upper, int* err_word);
// rounds: outer iterations of association + solve (cfg.outer_iters for every mapping and localising frame)
int map_register_device(aloam_ctx* c, int nb, const MapLaneIO* io, int nq_upper, int rounds, const PriorSearch* prior = nullptr);
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
// a finished group handed to the context: released by aloam_destroy
inline void own(aloam_ctx* c, BufGroup&& g) {
  BufGroup* q = new BufGroup(std::move(g));
  own(c, [q] { delete q; });
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

// S: LmSummary, or the LmHead of a recorded row (the same fields)
template <typename S>
void fill_stats_from(const S* h_summary, aloam_stats* st, int outer, int flags, float ms) {
  if (!st) return;
  std::memset(st, 0, sizeof(*st));
  st->flags = flags;
  st->ms_total = ms;
  for (int it = 0; it < outer && it < 4; ++it) {
    const S& s = h_summary[it];
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
// the stats of one scan-to-map frame (aloam_mapper_step, and the rows of the mapped stream calls): a frame that skipped its
// optimisation on a thin map has zeroed stats and only its flags; any other, its outer iterations' summaries
template <typename S>
void frame_stats_from(const S* summary, aloam_stats* st, int outer, int flags, float ms) {
  if (!(flags & ALOAM_FLAG_MAP_TOO_THIN)) { fill_stats_from(summary, st, outer, flags, ms); return; }
  if (!st) return;
  std::memset(st, 0, sizeof(*st));
  st->flags = flags;
  st->ms_total = ms;
}

int check_view(const aloam_cloud_view& v) {
  if (v.n < 0) return ALOAM_ERR_INVALID_ARG;
  if (v.n > 0 && (!v.data || (v.stride_floats != 4 && v.stride_floats != 8))) return ALOAM_ERR_INVALID_ARG;
  return ALOAM_OK;
}

}  // namespace
