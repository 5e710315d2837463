// Kernel declarations shared between the .cu translation units and the host-side context (capi.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include "common.cuh"

#define ALOAM_MAX_RING 4096                  // == ALOAM_MAX_RING_POINTS of the public header
#define ALOAM_ERR_RING_TOO_LARGE_DEV (-7)    // == ALOAM_ERR_RING_TOO_LARGE
#define ALOAM_LM_THREADS 288
#define ALOAM_LM_MAX_TRACE 8
#define ALOAM_N_KERNEL_IDS 32

namespace aloam {

// ---- batching: one launch covers up to ALOAM_MAX_BATCH independent trajectories ("lanes").  Every per-trajectory
// kernel takes its arguments as a by-value array indexed by blockIdx.y (or .z / .x where noted); a single trajectory is
// the batch of one.  __grid_constant__ keeps the array in the constant bank (no local copy for the dynamic index).
#ifndef ALOAM_MAX_BATCH
#define ALOAM_MAX_BATCH 16   // == the public header
#endif
template <typename T> struct Batch { T a[ALOAM_MAX_BATCH]; };

// ---- features.cu
size_t ring_features_smem_bytes(int max_ring, bool merge);   // merge: the 512-thread kernel (second key buffer)
void features_debug_cycles(long long* host64x8);   // 65 rows of 8 + 12: per-ring phase stamps, pick-walk stamps of ring 8
void features_debug_enable(int on);
struct ClassifyArgs { const float* raw; int n, stride; int8_t* ring_out; int* hist; ScanScalars* sc; };
struct RingScanArgs { const float* raw; int stride, nblocks; const int* hist; int* offsets; int* ring_start; int* scan_start; int* scan_end;
                      ScanScalars* sc; ScanScalars* sc_next; int* n_full_out; };
struct ScatterArgs { const float* raw; int n, stride; const int8_t* ring_in; const int* offsets; const ScanScalars* sc; Pt4* full; };
struct RingFeatArgs { const Pt4* full; const int* ring_start; Pt4 *st_sharp, *st_less_sharp, *st_flat, *st_less_flat; int* st_counts;
                      float* dbg_curv; int8_t* dbg_label; ScanScalars* sc; };
struct CompactArgs { const Pt4 *st_sharp, *st_less_sharp, *st_flat, *st_less_flat; const int* st_counts; Pt4 *sharp, *less_sharp, *flat, *less_flat;
                     int* counts; int *rs_ls, *rs_lf; };
__global__ void k_classify(const __grid_constant__ Batch<ClassifyArgs> B, int n_scans, float thres2);          // grid (blocks, lanes)
__global__ void k_ring_scan(const __grid_constant__ Batch<RingScanArgs> B, int n_scans);                       // grid (lanes)
__global__ void k_scatter(const __grid_constant__ Batch<ScatterArgs> B);                                       // grid (blocks, lanes)
__global__ void k_ring_features(const __grid_constant__ Batch<RingFeatArgs> B, int n_scans, float leaf, int max_ring);        // grid (2 * rings, 1), clusters of 2 CTAs x 512 threads
__global__ void k_ring_features_batch(const __grid_constant__ Batch<RingFeatArgs> B, int n_scans, float leaf, int max_ring);  // same, 256 threads (batches)
__global__ void k_compact(const __grid_constant__ Batch<CompactArgs> B, int n_scans, int max_ring);           // grid (rings, lanes)

// ---- odometry.cu
// (azimuth bucket x ring) index over one cloud = what replaces a kd-tree build (laserOdometry.cpp:567-568)
#define ALOAM_NB 128   // azimuth buckets (2.8 deg)
struct RabIndex {
  int* cnt;         // [NB*64] scratch counters (left zeroed by k_rab_scan)
  int* start;       // [NB*64 + 1] first slot of cell (bucket*64 + ring) in gpts
  int* cell_of;     // [capacity] cell of point i
  int* rank_of;     // [capacity] rank of point i inside its cell
  float4* gpts;     // [capacity] cell-contiguous copy: x, y, z, bits(ring << 24 | original index)
};
struct LastCloud {
  const Pt4* pts;   // the cloud in its original (ring-major) order
  const int* n;     // device scalar: number of points
  RabIndex index;
};
__global__ void k_ring_offsets(const Pt4* pts, int n, int* ring_start, int* err);
struct RabArgs { RabIndex a; const Pt4* pa; const int* na; RabIndex b; const Pt4* pb; const int* nb; };
__global__ void k_rab_count(const __grid_constant__ Batch<RabArgs> B);   // grid (blocks, 2 clouds, lanes)
__global__ void k_rab_scan(const __grid_constant__ Batch<RabArgs> B);    // grid (2 clouds, lanes)
__global__ void k_rab_fill(const __grid_constant__ Batch<RabArgs> B);    // grid (blocks, 2 clouds, lanes)

// one residual block, ready for the LM kernel (doubles; built once per association like the Ceres cost functions)
struct __align__(8) BlockRec {
  double cp[3];  // curr_point (untransformed)
  double a[3];   // edge: last_point_a          plane: last_point_j      plane-norm: unit normal
  double b[3];   // edge: last_point_b          plane: ljm_norm          plane-norm: unused
  double s;      // edge / plane: interpolation ratio s of the functor (1 unless DISTORTION)     plane-norm: negative_OA_dot_norm
  double w;      // edge: 1 / |a-b| (1 / de.norm())
  int type;      // 0 edge, 1 plane, 2 plane-norm, -1 = no residual (query without correspondence)
  int pad;
};
#define ALOAM_MAX_QUERIES 16384   // capacity of the sharp / flat query buffers (ctx.h kMaxQueries)
struct OdomParams { double dist_sq_thresh; double nearby_scan; int distortion; /* laserOdometry.cpp:59 #define DISTORTION */ };
__global__ void k_transform_to_end(const Pt4* in, int n, const double* pose7, int distortion, Pt4* out);
struct AssocArgs { const Pt4* sharp; const Pt4* flat; const int* feat_counts /*[4]*/; LastCloud corner, surf; const double* pose7;
                   BlockRec* blocks; int* corr /*[(n_sharp+n_flat)][4] a,b,c,valid ; may be null*/; };
__global__ void k_odom_assoc(const __grid_constant__ Batch<AssocArgs> B, OdomParams prm, int max_sharp);   // grid (query groups, lanes)
__global__ void k_knn_last(LastCloud cloud, const Pt4* queries, int nq, int* idx, float* sqd);

// ---- mapping.cu
// hash grid over a map cloud = what replaces the kd-tree builds of laserMapping.cpp:558-559
struct GridDyn {   // device-resident: everything about the indexed cloud that the kernels need and the host may not know
  int n;           // points in the cloud
  unsigned mask;   // table size - 1 (power of two >= 1.25 n)
  int cursor;      // storage cursor of k_grid_alloc
  int owned;       // sharded: points in cells this rank owns (halo excluded)
};
struct GridTable {
  uint4* slots;      // [cap_slots] one 16-byte word per slot: {cell key lo, hi (~0 = empty), points in the cell, end of its slice in gpts}
  GridDyn* dyn;
  float4* gpts;      // [capacity] cell-contiguous copy: x, y, z, bits(original index)
  unsigned cap_slots;
  float cs, inv_cs;  // cell edge [m]
};
struct MapCloud { GridTable grid; };
unsigned grid_mask_for(int n, unsigned cap_slots);
// the mapper's index build and association run over all lanes of aloam_scan_stream_mapped_batch at once: every kernel takes
// one record per lane and finds its own in blockIdx.z (the host API is the batch of one)
struct GridArgs { GridTable a; const Pt4* pa; const int* na; GridTable b; const Pt4* pb; const int* nb; };   // corner, surf
__global__ void k_grid_setup(const __grid_constant__ Batch<GridArgs> B);    // na / nb -> GridDyn
__global__ void k_grid_clear(const __grid_constant__ Batch<GridArgs> B);
__global__ void k_grid_insert(const __grid_constant__ Batch<GridArgs> B, int shard_rank, int shard_count);
__global__ void k_grid_alloc(const __grid_constant__ Batch<GridArgs> B);
__global__ void k_grid_fill(const __grid_constant__ Batch<GridArgs> B);
// 5-NN (warp per stack point) then line / plane fit + residual block (thread per stack point), laserMapping.cpp:577-687;
// counts3 = {n_corner, n_surf, total} in device memory, queries = corner then surf
struct MapAssocArgs { const Pt4* corner_stack; const Pt4* surf_stack; const int* counts3; MapCloud corner_map, surf_map; const double* pose7;
                      float4* nbr; BlockRec* blocks; double* fits; };
__global__ void k_map_knn5(const __grid_constant__ Batch<MapAssocArgs> B, int shard_rank, int shard_count);
__global__ void k_map_fit(const __grid_constant__ Batch<MapAssocArgs> B);
__global__ void k_map_knn(MapCloud map, const Pt4* queries, int nq, int k, int* idx, float* sqd);

// ---- voxel.cu: segmented, device-resident pcl::VoxelGrid (aloam_voxel_filter, the scan-stack filters and the per-cube re-filter
// of the mapping loop)
#define ALOAM_MAX_SEGS 160
struct SegDesc { const Pt4* src; const int* n_in; float leaf; Pt4* dst; int* n_out; };
struct SegFilter {
  const SegDesc* seg;   // [n_seg] device
  const int* n_seg;     // device
  int* off;             // [MAX_SEGS + 1] compact offsets of the segments
  int* rank0;           // [MAX_SEGS + 1] voxels before each segment
  int* bbox;            // [MAX_SEGS][6] ordered-int min / max
  int* total;           // points over all segments
  int* pass;            // [MAX_SEGS] 1: the segment is returned unchanged (index overflow), set for every non-empty segment
  int* err;             // sticky error word (bit 0: a segment needs more than idx_bits index bits)
  int idx_bits;         // bits of the voxel index inside a segment, 1 .. 32 (32: one segment, the key is PCL's int index)
  int seg0, seg_cap;    // this pass handles segments seg0 .. seg0 + seg_cap - 1 (as many as fit beside idx_bits in a 32-bit key)
};
// everything one segmented filter owns on the device (vox_seg_alloc); its calls run one after another on one stream
struct SegBuffers {
  SegDesc* segs = nullptr;   // [MAX_SEGS]
  int* n_seg = nullptr;
  int *off = nullptr, *rank0 = nullptr, *bbox = nullptr, *total = nullptr, *pass = nullptr;   // see SegFilter
  unsigned* keys[2] = {nullptr, nullptr};
  int* vals[2] = {nullptr, nullptr};
  int *hist = nullptr, *block_heads = nullptr, *heads_total = nullptr;   // heads_total: k_vox_blockscan's voxel count (not read)
  Pt4* tmp = nullptr;
  size_t cap = 0;            // points over all segments of one call
  int coop_grid = 1;         // CTAs of the cooperative radix sort: one per SM of the context's device
};
inline SegFilter seg_filter(const SegBuffers& b, int idx_bits, int* err) {
  return SegFilter{b.segs, b.n_seg, b.off, b.rank0, b.bbox, b.total, b.pass, err, idx_bits, 0, ALOAM_MAX_SEGS};
}
// one lane of a segmented-filter launch over several lanes (the mapper's lanes each own a SegBuffers): the filter and its sort
// buffers; every kernel of voxel.cu takes one per lane and finds its own in blockIdx.z
struct VoxLane { SegFilter f; unsigned* keys[2]; int* vals[2]; int* hist; int* block_heads; int* heads_total; Pt4* tmp; };

// ---- lm.cu
struct LmParams {
  int max_iters;
  double huber_a;
  double initial_radius, max_radius, min_radius;
  double min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
  double function_tolerance, gradient_tolerance, parameter_tolerance;
  int max_invalid;
};
struct LmSummary {
  int termination, num_iterations, num_successful, num_jac_evals;
  int n_edge, n_plane;      // residual blocks by kind
  double initial_cost, final_cost;
  int trace_rows; int pad;
  long long cyc_total, cyc_eval, cyc_chol, cyc_plus, cyc_grad;   // SM clock cycles (thread 0 of CTA 0): whole solve / evaluation passes / trust-region steps / residual blocks of the thread / cluster barriers
  double trace[ALOAM_LM_MAX_TRACE][8];
};
// mode 0: full trust-region solve, x updated in place ; mode 1: one evaluation, out28 = [JtJ upper 21, g 6, cost]
// integrate != 0 : after the solve compose the world pose (laserOdometry.cpp:504-505): world7 <- world7 (+) x
struct LmArgs { const BlockRec* blocks; const int* n_blocks_ptr; int n_blocks_host; double* x7; LmSummary* summary; double* out28; double* world7; };
// Sharded solve over NVLink peer memory (multi-GPU scan-to-map, comm.cu): every rank's LM cluster stores its 32 partial sums,
// each 8-byte word tagged with the evaluation's sequence number, into a mailbox in EVERY rank's memory (peer stores through
// NVSwitch), polls its own mailbox until every rank's words carry the tag and adds the contributions in rank order -- the
// all-reduce of the normal equations happens INSIDE the solve kernel, one launch per solve, no kernel boundary around the
// 256-byte exchange.  world 0: no exchange; world 1 (never a real job: aloam_comm_init keeps a one-rank world off the sharded
// path) is the loopback of a context emulating a rank.
#define ALOAM_MAX_RANKS 16
struct PeerX {
  double* box[ALOAM_MAX_RANKS];             // mailbox of rank r: [2 parities][world][32][2] 8-byte words {payload half, tag} (peer-mapped device memory)
  unsigned long long* seq;                  // this rank's evaluation counter (device), identical on all ranks by construction
  double* gtot;                             // [2][32] this rank's summed totals (local)
  int* err;                                 // set to 1 when a peer did not answer in time
  int rank, world;
};
__global__ void k_lm_solve(const __grid_constant__ Batch<LmArgs> B, LmParams prm, int mode, int integrate);   // every block s == 1, one GPU; grid (8, lanes), clusters of 8 along x
__global__ void k_lm_solve_x(const __grid_constant__ Batch<LmArgs> B, LmParams prm, int mode, int integrate, const __grid_constant__ PeerX px);   // general s and / or peer exchange
// sharded solve: per-evaluation kernels around an ncclAllReduce (see lm.cu, comm.cu)
size_t lm_state_bytes();
size_t lm_dynamic_smem_bytes();   // dynamic shared memory of k_lm_solve / k_lm_eval_shard (opt-in > 48 KB)
__global__ void k_lm_eval_shard(const BlockRec* blocks, const int* n_ptr, int n_host, const double* x7, void* state, int first, double huber_a, double* local32);
__global__ void k_lm_tr_shard(void* state, const double* tot32, double* x7, int first, LmParams prm, LmSummary* summary);
// packs API-side residual blocks (11 doubles) into BlockRec
__global__ void k_pack_blocks(const double* packed, int n, BlockRec* out);

}  // namespace aloam
