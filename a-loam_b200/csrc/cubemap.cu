// Map cube store of alaserMapping and the per-frame loop around it -- replaces laserMapping.cpp:74-108 (state),
// :142-163 (pose hand-off, pointAssociateToMap), :309-550 (centre cube, ring-buffer shift, 75-cube gather, stack
// filters) and :736-801 (insertion, per-cube VoxelGrid).  SURVEY.md section 8 f-1 / f-2.
//
// Second version: the WHOLE frame runs on the device without a host synchronisation, so it can sit at the end of the scan
// stream (aloam_scan_stream_mapped) or behind the host API (aloam_mapper_step, one sync at the end to return the pose):
//   * state (T_wmap_wodom, centre offsets, cube -> run table, per-run counts and orders, slab occupancy bitmaps) lives in device memory;
//   * k_mapper_begin : transformAssociateToMap, centre cube, ring-buffer shift (the reference rotates 4851 smart pointers;
//                      here one CTA permutes the cube -> run table, one thread per line of cubes, and frees the runs of
//                      the cubes that scroll out), valid-cube list in the reference's i, j, k order;
//   * k_mapper_gather: the <= 75 valid cubes device-to-device into the submap, then the hash-grid build of mapping.cu;
//   * the two scan-stack filters as ONE segmented VoxelGrid (voxel.cu), the registration of mapping.cu on device views;
//   * k_mapper_update: transformUpdate, refined pose out;
//   * k_cube_ids / k_cube_insert: pointAssociateToMap + cube of the stored point, then a count pass, the runs every cube
//                      needs (a new cube's first run, a grown cube's larger one, in the order of their first stack point),
//                      the move of grown cubes, and a STABLE append (push_back order = stack order): one CTA walks the
//                      stack in chunks, warps take turns, __match_any groups the lanes of a cube and the group leader
//                      advances the cube's running end -- O(n) instead of the O(n^2 / 256) rank search of the first version;
//   * the per-cube re-filter of the valid cubes as ONE segmented VoxelGrid over up to 150 segments, in place.
//   * the published clouds (:806-848): k_export_sizes lays a lane's store out in the reference's order and k_store_copy copies it
//                      (aloam_mapper_export), k_register_full moves a mapped scan's full cloud by the frame's refined pose.
//   * localisation against a prior map (aloam_prior_map_load, aloam_lane_localise): the store of a saved lane, frozen, packed in
//                      cube order and indexed ONCE with the hash grid of mapping.cu; a localising lane's frame is k_locate_begin
//                      (hand-off, centre cube, clipped 5 x 5 x 3 window -- no shift), the stack filters, the registration of
//                      mapping.cu through k_map_knn5_prior, k_mapper_update: no gather, no index build, no insertion, no re-filter.
// Slabs are a POOL (1024 per cloud type, 16 k corner / 64 k surf points each: 1.3 GB) handed out on the device on first
// insertion, not 4851 x 2 slabs (6.4 GB) up front.  A cube holds an aligned RUN of 2^k slabs (k = 0 while its lane's cube
// growth is off, aloam_set_cube_growth); with growth on a cube whose run fills moves to the smallest run that holds its new
// count, up to ALOAM_MAX_CUBE_POINTS.  A cube at its ceiling or a run that cannot be found drops the overflow and raises
// ALOAM_FLAG_CUBE_OVERFLOW instead of failing the frame (the reference grows its cubes without bound between re-filters).
#include <climits>
#include <memory>
#include "common.cuh"
#include "ctx.h"
#include "grid.cuh"
#include "quat.cuh"

namespace {

constexpr int CW = 21, CH = 21, CD = 11, NCUBE = CW * CH * CD;   // laserCloudWidth / Height / Depth (:77-82)
constexpr int kMaxValid = 128;
constexpr int kPool = 1024;                                      // physical slabs per cloud type
constexpr int kPoolWords = kPool / 32;                           // words of a type's occupancy bitmap
constexpr int kMaxOrder = 10;                                    // a run of 2^10 slabs is the whole pool
static_assert(NCUBE == kSnapCubes && kMaxValid == kSnapValid && kPool == kSnapPool, "the snapshot format describes this store");
constexpr int kExportSegs = 2 * NCUBE;                           // segments of an export: segment 2 v + t is type t of its v-th cube

}  // namespace

// Where the points of an export are (device memory): segment s < nseg sits at positions [off[s], off[s + 1]) of the export and
// at base[s] in the store, which may be a lane's slab or a cube of the prior map; total = off[nseg]
struct aloam::ExportLayout {
  int nseg;
  long long total;
  long long off[kExportSegs + 1];
  Pt4* base[kExportSegs];
};

namespace {

struct MapperState {
  double q_wmap_wodom[4], t_wmap_wodom[3];   // :116-117
  double x[7];                               // parameters[7] of this frame: q_w_curr (xyzw), t_w_curr
  double q_wodom[4], t_wodom[3];             // odometry pose of this frame
  int cen[3];                                // laserCloudCenWidth / Height / Depth (:74-76)
  int ctr[3];                                // centerCubeI / J / K after the shift
  int n_valid;
  int valid[kMaxValid];                      // laserCloudValidInd (i + 21 j + 441 k) in the reference's loop order
  int sub_off[2][kMaxValid + 1];
  int n_sub[2];                              // gathered submap sizes (corner, surf)
  int stack_counts[4];                       // filtered stack sizes: corner, surf, total used by the registration, raw total
  int in_counts[2];                          // sizes of the incoming less-sharp / less-flat clouds (host API path)
  int flags;                                 // ALOAM_FLAG_* of this frame
  int frame_err;                             // `err` of the last completed frame (read back with `flags`)
  int err;                                   // of the running frame -- bit 0: voxel index range, bit 1: a cube at its capacity
                                             // dropped points, bit 2: no free run, bit 3: submap capacity, bit 4: cubes left out
                                             // of the re-filter (its buffer); cleared when the frame ends
  int err_acc;                               // OR of the frames' words over one aloam_scan_stream_mapped call
  int frames;
  int zero, sink;                            // always 0 (count of a cube without a slab) ; write-only dummy
  int max_ord[2];                            // the largest run of the lane's store per type is 2^max_ord slabs: 0 with cube
                                             // growth off, fixed at the trajectory's start
  unsigned used[2][kPoolWords];              // slab occupancy per type: bit s of word s / 32 is set while slab s is in a run
  int slab_of[2][NCUBE];                     // cube -> first slab of its run of that type, -1 = none
  int cnt[2][kPool];                         // points of the run that starts at a slab
  unsigned char ord[2][kPool];               // the run that starts at a slab holds 2^ord slabs
};

}  // namespace

// What a scan-to-map frame runs on, mapping or localising: the frame state on the device and its pinned mirror (debug / host API
// read-back), the registration set and the segmented filter of the stack filters.  Every kernel of a frame takes the state the same
// way for both modes; a localising frame leaves the slab tables unused and keeps its window tables in sub_off.  The frame owns its
// buffers in `mem`, except lane 0 of the mapper, which registers with the context's set c->map, shared with the host API.
struct aloam::LaneFrame {
  BufGroup mem;
  MapperState* d_state = nullptr;
  MapperState* h_state = nullptr;
  MapReg* reg = nullptr;   // &set, or the context's set
  MapReg set = {};
  SegBuffers buf;
};

// A lane's cube store: its frame (whose filter also runs the per-cube re-filter) and the store's buffers, in `mem`
struct aloam::Mapper {
  LaneFrame frame;
  BufGroup mem;
  int cap[2] = {0, 0};
  Pt4* d_pts[2] = {nullptr, nullptr};       // [kPool * cap] slabs
  Pt4* d_sub[2] = {nullptr, nullptr};       // gathered submap
  Pt4* d_in[2] = {nullptr, nullptr};        // host API: uploaded less-sharp / less-flat clouds
  Pt4* d_world = nullptr;                   // insertion scratch: transformed stack points
  int* d_cube = nullptr;                    //                    their cube index (-1 = outside the ring buffer)
  double* d_pose_io = nullptr;              // [14] host API: odometry pose in, refined pose out
  // aloam_debug_seg_voxel_filter, created on first use: segments back to back [frame.buf.cap], their sizes [ALOAM_MAX_SEGS] and a
  // private error word, one group
  BufGroup dbg;
  Pt4* d_dbg_pts = nullptr;
  int* d_dbg_counts = nullptr;
  int* d_dbg_err = nullptr;
  int max_sub = 0;
};

// The prior map: the store of a mapped lane snapshot, frozen.  Per cloud type the points packed in cube order (cube_start = the
// exclusive prefix of the snapshot's counts) and a hash grid over ALL of them, built once by prior_index; the centre offsets of
// the store, which never change (no localising frame shifts the ring buffer); the layout of its ALOAM_EXPORT_MAP export.  Its
// buffers, the digest's included, are one group, freed with the map by prior_map_release.
struct aloam::PriorMap {
  BufGroup mem;
  Pt4* pts[2] = {nullptr, nullptr};
  int n[2] = {0, 0};
  int cen[3] = {0, 0, 0};
  int* d_cube_start = nullptr;   // [2][NCUBE + 1]
  int* d_n = nullptr;            // [2]
  GridTable grid[2] = {};
  ExportLayout* d_layout = nullptr;
  // per type, from the cube table: the largest cube, the cubes that hold points and the slabs their runs take with cube growth
  // on -- whether a lane store can hold a copy of the map (aloam_lane_map_on_prior)
  int max_cube[2] = {0, 0}, n_cubes[2] = {0, 0}, run_slabs[2] = {0, 0};
  // aloam_prior_map_digest: computed by the first call that needs it (k_prior_digest), kept until the map is released
  bool have_digest = false;
  unsigned long long digest = 0;
  unsigned long long* d_digest = nullptr;
};

namespace {

// what every kernel of a frame needs of one lane: the frame runs over all lanes at once, each launch taking one record per lane
// (lane = blockIdx.z)
struct MapperLane {
  MapperState* S;
  const double* odom7;   // odometry pose of this scan
  double* out7;          // refined pose out (may be null)
  Pt4* pts[2];           // slab pools
  int cap[2];
  Pt4* sub[2];           // gathered submap
  const Pt4* in[2];      // less-sharp / less-flat clouds of the scan and their sizes
  const int* n_in[2];
  Pt4* stack[2];         // filtered stacks
  Pt4* world;            // insertion scratch
  int* cube;
  SegDesc* segs;         // the lane's segmented filter
  int* n_seg;
};

// int((v + 25.0) / 50.0) + centre, minus one when v + 25.0 < 0   (:314-325, :741-750)
__host__ __device__ inline int cube_coord(double v, int centre) {
  int c = int((v + 25.0) / 50.0) + centre;
  if (v + 25.0 < 0) c--;
  return c;
}
__host__ __device__ inline int cube_index(int i, int j, int k) { return i + CW * j + CW * CH * k; }

// the slabs of the run of 2^o slabs that starts at slab s: the bits of the occupancy bitmap `used` they cover.  Word w's mask.
__host__ __device__ inline unsigned run_mask(int s, int o, int w) {
  const int n = 1 << o;
  if (n >= 32) return w >= (s >> 5) && w < ((s + n) >> 5) ? ~0u : 0u;
  return w == (s >> 5) ? ((1u << n) - 1u) << (s & 31) : 0u;
}

// :327-509 -- one step of the ring buffer along `axis` for the line (u, v) of this thread; towards_high: every cube moves one
// index up, the top cube wraps to index 0 and is emptied (its run goes back to the pool)
__device__ void rotate_line(MapperState* S, int axis, bool towards_high, int u, int v) {
  const int n[3] = {CW, CH, CD};
  const int a = axis, b = (axis + 1) % 3, cc = (axis + 2) % 3;
  auto at = [&](int t) { int ijk[3]; ijk[a] = t; ijk[b] = u; ijk[cc] = v; return cube_index(ijk[0], ijk[1], ijk[2]); };
#pragma unroll
  for (int ty = 0; ty < 2; ++ty) {
    int* so = S->slab_of[ty];
    int wrapped;
    if (towards_high) {
      wrapped = so[at(n[a] - 1)];
      for (int t = n[a] - 1; t >= 1; --t) so[at(t)] = so[at(t - 1)];
      so[at(0)] = -1;
    } else {
      wrapped = so[at(0)];
      for (int t = 0; t < n[a] - 1; ++t) so[at(t)] = so[at(t + 1)];
      so[at(n[a] - 1)] = -1;
    }
    if (wrapped >= 0) {
      S->cnt[ty][wrapped] = 0;
      const int o = S->ord[ty][wrapped];
      for (int w = wrapped >> 5; w < kPoolWords; ++w) {   // other lines free other runs of the same words
        const unsigned m = run_mask(wrapped, o, w);
        if (!m) break;
        atomicAnd(&S->used[ty][w], ~m);
      }
    }
  }
}

// the state of a fresh trajectory (laserMapping.cpp:74-117): identity T_wmap_wodom, centre cube (10, 10, 5), every slab free
// and no cube holding one, runs of up to 2^ord0 corner / 2^ord1 surf slabs.  Run by all threads of one CTA.  It leaves alone the word of the call (err_acc) and every field the
// stack filter writes while k_mapper_begin runs beside it (stack_counts, err, in_counts): between frames `err` is 0 already
// (k_mapper_finish), and reset_lane zeroes the whole state before it runs this.
__device__ void mapper_fresh_state(MapperState* S, int ord0, int ord1) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = tid; i < NCUBE; i += nt) { S->slab_of[0][i] = -1; S->slab_of[1][i] = -1; }
  for (int i = tid; i < kPool; i += nt) { S->cnt[0][i] = 0; S->cnt[1][i] = 0; S->ord[0][i] = 0; S->ord[1][i] = 0; }
  for (int i = tid; i < 2 * kPoolWords; i += nt) S->used[i / kPoolWords][i % kPoolWords] = 0u;
  for (int i = tid; i < kMaxValid; i += nt) S->valid[i] = 0;
  for (int i = tid; i < 2 * (kMaxValid + 1); i += nt) S->sub_off[i / (kMaxValid + 1)][i % (kMaxValid + 1)] = 0;
  if (tid == 0) {
    for (int k = 0; k < 4; ++k) { S->q_wmap_wodom[k] = k == 3 ? 1.0 : 0.0; S->q_wodom[k] = 0.0; }
    for (int k = 0; k < 3; ++k) { S->t_wmap_wodom[k] = 0.0; S->t_wodom[k] = 0.0; S->ctr[k] = 0; }
    for (int k = 0; k < 7; ++k) S->x[k] = 0.0;
    S->cen[0] = 10; S->cen[1] = 10; S->cen[2] = 5;
    S->n_valid = 0; S->n_sub[0] = 0; S->n_sub[1] = 0;
    S->flags = 0; S->frame_err = 0; S->frames = 0; S->zero = 0; S->sink = 0;
    S->max_ord[0] = ord0; S->max_ord[1] = ord1;
  }
}
// grid (1): the host-side reset of one lane (reset_lane)
__global__ void __launch_bounds__(1024) k_mapper_reset(MapperState* S, int ord0, int ord1) { mapper_fresh_state(S, ord0, ord1); }

// transformAssociateToMap (:142-146): x = T_wmap_wodom * odometry pose -- also the high-frequency pose of :214-215
__device__ __forceinline__ void associate_to_map(const MapperState* S, const double* odom7, double* x) {
  const Qd qm{S->q_wmap_wodom[0], S->q_wmap_wodom[1], S->q_wmap_wodom[2], S->q_wmap_wodom[3]};
  const Qd qo{odom7[0], odom7[1], odom7[2], odom7[3]};
  const double to[3] = {odom7[4], odom7[5], odom7[6]};
  const Qd q0 = qmul(qm, qo);
  double r[3]; qrot(qm, to, r);
  x[0] = q0.x; x[1] = q0.y; x[2] = q0.z; x[3] = q0.w;
  x[4] = r[0] + S->t_wmap_wodom[0]; x[5] = r[1] + S->t_wmap_wodom[1]; x[6] = r[2] + S->t_wmap_wodom[2];
}

// transformAssociateToMap (:142-146), centre cube + shift (:314-509), valid cubes (:511-529), gather offsets
__device__ __forceinline__ void mapper_begin_body(MapperState* S, const double* __restrict__ odom7, int max_sub, bool fresh, int ord0, int ord1) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (fresh) {   // the lane starts a new trajectory with this frame: no extra launch, in order on the mapper stream
    mapper_fresh_state(S, ord0, ord1);
    __syncthreads();
  }
  __shared__ int s_ctr[3], s_cen[3];
  const int tid = threadIdx.x;
  if (tid == 0) {
    const Qd qo{odom7[0], odom7[1], odom7[2], odom7[3]};
    const double to[3] = {odom7[4], odom7[5], odom7[6]};
    associate_to_map(S, odom7, S->x);
    S->q_wodom[0] = qo.x; S->q_wodom[1] = qo.y; S->q_wodom[2] = qo.z; S->q_wodom[3] = qo.w;
    S->t_wodom[0] = to[0]; S->t_wodom[1] = to[1]; S->t_wodom[2] = to[2];
    for (int a = 0; a < 3; ++a) { s_cen[a] = S->cen[a]; s_ctr[a] = cube_coord(S->x[4 + a], S->cen[a]); }
    S->flags = 0;
  }
  __syncthreads();
  const int dims[3] = {CW, CH, CD};
  for (int a = 0; a < 3; ++a) {
    const int nb = dims[(a + 1) % 3], nc = dims[(a + 2) % 3];
    for (;;) {   // :327-416 pattern: shift up while the centre is within 3 cubes of the low edge
      const int ctr = s_ctr[a];
      __syncthreads();
      if (!(ctr < 3)) break;
      if (tid < nb * nc) rotate_line(S, a, true, tid % nb, tid / nb);
      __syncthreads();
      if (tid == 0) { s_ctr[a]++; s_cen[a]++; }
      __syncthreads();
    }
    for (;;) {   // shift down while it is within 3 cubes of the high edge
      const int ctr = s_ctr[a];
      __syncthreads();
      if (!(ctr >= dims[a] - 3)) break;
      if (tid < nb * nc) rotate_line(S, a, false, tid % nb, tid / nb);
      __syncthreads();
      if (tid == 0) { s_ctr[a]--; s_cen[a]--; }
      __syncthreads();
    }
  }
  __shared__ int s_valid[kMaxValid], s_n[2][kMaxValid], s_nv;
  if (tid == 0) {
    for (int a = 0; a < 3; ++a) { S->cen[a] = s_cen[a]; S->ctr[a] = s_ctr[a]; }
    int nv = 0;
    for (int i = s_ctr[0] - 2; i <= s_ctr[0] + 2; ++i)
      for (int j = s_ctr[1] - 2; j <= s_ctr[1] + 2; ++j)
        for (int k = s_ctr[2] - 1; k <= s_ctr[2] + 1; ++k)
          if (i >= 0 && i < CW && j >= 0 && j < CH && k >= 0 && k < CD) s_valid[nv++] = cube_index(i, j, k);
    s_nv = nv;
    S->n_valid = nv;
  }
  __syncthreads();
  const int nv = s_nv;
  if (tid < 2 * nv) {   // the counts of the valid cubes, all loads in flight at once
    const int ty = tid >= nv, v = ty ? tid - nv : tid;
    const int s = S->slab_of[ty][s_valid[v]];
    s_n[ty][v] = s < 0 ? 0 : S->cnt[ty][s];
    if (ty == 0) S->valid[v] = s_valid[v];
  }
  __syncthreads();
  if (tid < 2) {
    const int ty = tid;
    int off = 0;
    for (int v = 0; v < nv; ++v) {
      S->sub_off[ty][v] = off;
      int n = s_n[ty][v];
      if (off + n > max_sub) { n = max_sub - off; atomicOr(&S->err, 8); }   // submap capacity: truncated, flagged
      off += n;
    }
    S->sub_off[ty][nv] = off;
    S->n_sub[ty] = off;
  }
}
// grid (1, 1, lanes); bit l of `fresh`: record l starts a new trajectory with this frame, its state is reset first, with runs of
// up to 2^ord0 / 2^ord1 slabs (the context's cube growth)
__global__ void __launch_bounds__(1024) k_mapper_begin(const __grid_constant__ Batch<MapperLane> B, int max_sub, unsigned fresh, int ord0, int ord1) {
  const MapperLane& a = B.a[blockIdx.z];
  mapper_begin_body(a.S, a.odom7, max_sub, (fresh >> blockIdx.z) & 1u, ord0, ord1);
}

// grid (1, 1, lanes): the scans the mapper skips (mapping_skip_frame > 1) get the high-frequency pose of laserOdometryHandler
// (:197-229): T_wmap_wodom of the lane's latest mapper frame (queued before this kernel on the mapper stream) times the scan's
// odometry pose.  The cube store is not touched.
__global__ void k_mapper_high_freq(const __grid_constant__ Batch<MapperLane> B) {
  if (threadIdx.x) return;
  const MapperLane& a = B.a[blockIdx.z];
  double x[7];
  associate_to_map(a.S, a.odom7, x);
  for (int k = 0; k < 7; ++k) a.out7[k] = x[k];
}


// ---- localisation against a prior map: the frame of a lane that registers its scans against the context's frozen store

// one lane of k_locate_begin: its frame state, the scan's odometry pose, and for a lane that starts its trajectory with this
// frame (`fresh`) the T_wmap_wodom it starts from (aloam_lane_localise)
struct LocateLane {
  MapperState* S;
  const double* odom7;
  double init[7];
  int fresh;
};
// grid (1, 1, lanes), 256 threads: the head of a localising frame -- laserMapping.cpp:309-321 and :512-531 with the ring-buffer
// shift (:323-507) left out.  Pose hand-off as k_mapper_begin; centre cube from the prior map's fixed centre offsets `cen`; the
// valid list = the window's cubes inside the buffer, in the reference's loop order; and per type the window table
// S->sub_off[ty][w], w = (di + 2) * 15 + (dj + 2) * 3 + (dk + 1): the offset cube w's points would have in the gathered submap
// (exclusive scan of the window's counts in loop order), -1 for a cube outside the buffer.  cs = the prior map's cube prefix
// tables [2][NCUBE + 1].  n_sub feeds the thin-map test of k_mapper_prep.
__global__ void __launch_bounds__(256) k_locate_begin(const __grid_constant__ Batch<LocateLane> B, const int* __restrict__ cs, int cen0, int cen1, int cen2) {
  const LocateLane& a = B.a[blockIdx.z];
  MapperState* S = a.S;
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int tid = threadIdx.x;
  if (a.fresh) {
    mapper_fresh_state(S, 0, 0);   // (a locator's store tables stay unused)
    __syncthreads();
    if (tid < 4) S->q_wmap_wodom[tid] = a.init[tid];
    else if (tid < 7) S->t_wmap_wodom[tid - 4] = a.init[tid];
    __syncthreads();
  }
  __shared__ int s_ctr[3], s_cnt[2][ALOAM_WINDOW_CUBES];
  if (tid == 0) {
    associate_to_map(S, a.odom7, S->x);
    for (int k = 0; k < 4; ++k) S->q_wodom[k] = a.odom7[k];
    for (int k = 0; k < 3; ++k) S->t_wodom[k] = a.odom7[4 + k];
    const int cen[3] = {cen0, cen1, cen2};
    for (int k = 0; k < 3; ++k) { S->cen[k] = cen[k]; s_ctr[k] = cube_coord(S->x[4 + k], cen[k]); S->ctr[k] = s_ctr[k]; }
    S->flags = 0;
  }
  __syncthreads();
  if (tid < 2 * ALOAM_WINDOW_CUBES) {   // the counts of the window's cubes, all loads in flight at once
    const int ty = tid >= ALOAM_WINDOW_CUBES, w = ty ? tid - ALOAM_WINDOW_CUBES : tid;
    const int i = s_ctr[0] - 2 + w / 15, j = s_ctr[1] - 2 + (w / 3) % 5, k = s_ctr[2] - 1 + w % 3;
    int n = -1;
    if (i >= 0 && i < CW && j >= 0 && j < CH && k >= 0 && k < CD) { const int* t = cs + ty * (NCUBE + 1) + cube_index(i, j, k); n = t[1] - t[0]; }
    s_cnt[ty][w] = n;
  }
  __syncthreads();
  if (tid < 2) {
    const int ty = tid;
    int off = 0;
    for (int w = 0; w < ALOAM_WINDOW_CUBES; ++w) {
      const int n = s_cnt[ty][w];
      S->sub_off[ty][w] = n < 0 ? -1 : off;
      off += max(n, 0);
    }
    S->n_sub[ty] = off;
  } else if (tid == 32) {
    int nv = 0;
    for (int w = 0; w < ALOAM_WINDOW_CUBES; ++w)
      if (s_cnt[0][w] >= 0) S->valid[nv++] = cube_index(s_ctr[0] - 2 + w / 15, s_ctr[1] - 2 + (w / 3) % 5, s_ctr[2] - 1 + w % 3);
    S->n_valid = nv;
  }
}

// grid (1), 256 threads, after a memset of the state: the frame state of a localising lane restored from a format-2 snapshot
// (aloam_lane_restore) -- what a fresh localising START leaves before its first frame (k_locate_begin with `fresh`), with the
// saved T_wmap_wodom and the prior map's centre offsets.  A later frame reads only T_wmap_wodom of it; everything else it
// rewrites before reading.
struct Pose7 { double v[7]; };
__global__ void __launch_bounds__(256) k_locate_restore(MapperState* S, const __grid_constant__ Pose7 T, int cen0, int cen1, int cen2) {
  mapper_fresh_state(S, 0, 0);
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < 4; ++k) S->q_wmap_wodom[k] = T.v[k];
    for (int k = 0; k < 3; ++k) S->t_wmap_wodom[k] = T.v[4 + k];
    S->cen[0] = cen0; S->cen[1] = cen1; S->cen[2] = cen2;
  }
}

// the digest of a prior map (aloam_prior_map_digest, include/aloam_b200.h): sum over k of mix(k, w_k) mod 2^64 for the word
// sequence w = the three centre offsets, the cube-start tables cs[2][NCUBE + 1] (corner, then surf), the corner points, the surf
// points (4 float bit patterns each, packed cube order); every word a 32-bit pattern, zero-extended.  mix: splitmix64's finaliser
// of (k * golden gamma) ^ w.  Integer addition: the sum does not depend on how the words are split over threads.
__host__ __device__ inline unsigned long long digest_mix(unsigned long long k, unsigned w) {
  unsigned long long z = (k * 0x9E3779B97F4A7C15ull) ^ w;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
constexpr int kDigestThreads = 256;
constexpr int kDigestHead = 3 + 2 * (NCUBE + 1);   // words before the points
// grid-stride over the words, one 16-byte load per point; a warp-shuffle and shared-memory sum per CTA, one atomicAdd per CTA into
// *out (zeroed before)
__global__ void __launch_bounds__(kDigestThreads) k_prior_digest(int cen0, int cen1, int cen2, const int* __restrict__ cs, const float4* __restrict__ p0,
                                                                 int n0, const float4* __restrict__ p1, int n1, unsigned long long* __restrict__ out) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  unsigned long long s = 0;
  for (long long k = tid; k < kDigestHead; k += nt) {
    const unsigned w = k == 0 ? (unsigned)cen0 : k == 1 ? (unsigned)cen1 : k == 2 ? (unsigned)cen2 : (unsigned)__ldg(cs + (k - 3));
    s += digest_mix((unsigned long long)k, w);
  }
  const long long n = (long long)n0 + n1;
  for (long long i = tid; i < n; i += nt) {
    const float4 q = i < n0 ? __ldg(p0 + i) : __ldg(p1 + (i - n0));
    const unsigned long long k = kDigestHead + 4ull * (unsigned long long)i;
    s += digest_mix(k, __float_as_uint(q.x)) + digest_mix(k + 1, __float_as_uint(q.y)) + digest_mix(k + 2, __float_as_uint(q.z)) +
         digest_mix(k + 3, __float_as_uint(q.w));
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  __shared__ unsigned long long ws[kDigestThreads / 32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < kDigestThreads / 32 ? ws[threadIdx.x] : 0ull;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) atomicAdd(out, s);
  }
}

// grid (CTAs, 2 types): after the index build, every indexed point's packed index g (gpts.w, written by k_grid_fill) becomes
// prior_tag(cube i, j, k, rank in the cube): the cube is the last one whose prefix is <= g
__global__ void __launch_bounds__(256) k_prior_tag(const __grid_constant__ GridTable corner, const __grid_constant__ GridTable surf, const int* __restrict__ cs) {
  const GridTable& g = blockIdx.y == 0 ? corner : surf;
  const int* __restrict__ t = cs + blockIdx.y * (NCUBE + 1);
  const int n = g.dyn->n;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
    const int idx = __float_as_int(g.gpts[s].w);
    int lo = 0, hi = NCUBE;   // t[lo] <= idx < t[hi]
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (t[mid] <= idx) lo = mid; else hi = mid; }
    g.gpts[s].w = __uint_as_float(prior_tag(lo % CW, (lo / CW) % CH, lo / (CW * CH), idx - t[lo]));
  }
}


// grid (valid cubes, 2 types): slab -> submap (:531-539), device to device
__device__ __forceinline__ void mapper_gather_body(const MapperState* __restrict__ S, const Pt4* __restrict__ p0, const Pt4* __restrict__ p1,
                                                       int cap0, int cap1, Pt4* __restrict__ sub0, Pt4* __restrict__ sub1) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int v = blockIdx.x, ty = blockIdx.y;
  if (v >= S->n_valid) return;
  const int s = S->slab_of[ty][S->valid[v]];
  if (s < 0) return;
  const int off = S->sub_off[ty][v], n = S->sub_off[ty][v + 1] - off;
  const Pt4* __restrict__ src = (ty ? p1 : p0) + (size_t)s * (ty ? cap1 : cap0);
  Pt4* __restrict__ dst = (ty ? sub1 : sub0) + off;
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}
// grid (valid cubes, 2 types, lanes)
__global__ void __launch_bounds__(256) k_mapper_gather(const __grid_constant__ Batch<MapperLane> B) {
  const MapperLane& a = B.a[blockIdx.z];
  mapper_gather_body(a.S, a.pts[0], a.pts[1], a.cap[0], a.cap[1], a.sub[0], a.sub[1]);
}


// segment descriptors of the two scan-stack filters (:543-549)
__device__ __forceinline__ void seg_two_body(SegDesc* segs, int* n_seg, const Pt4* c_in, const int* nc, float c_leaf, Pt4* c_out, int* nc_out, const Pt4* s_in, const int* ns,
                          float s_leaf, Pt4* s_out, int* ns_out) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    segs[0] = SegDesc{c_in, nc, c_leaf, c_out, nc_out};
    segs[1] = SegDesc{s_in, ns, s_leaf, s_out, ns_out};
    *n_seg = 2;
  }
}
// grid (1, 1, lanes)
__global__ void k_seg_two(const __grid_constant__ Batch<MapperLane> B, float c_leaf, float s_leaf) {
  const MapperLane& a = B.a[blockIdx.z];
  seg_two_body(a.segs, a.n_seg, a.in[0], a.n_in[0], c_leaf, a.stack[0], &a.S->stack_counts[0], a.in[1], a.n_in[1], s_leaf, a.stack[1], &a.S->stack_counts[1]);
}


// after the stack filters: the map-too-thin test of :554 (on the gathered submap) -> number of queries the registration sees
__device__ __forceinline__ void mapper_prep_body(MapperState* S) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x || blockIdx.x) return;
  const int total = S->stack_counts[0] + S->stack_counts[1];
  S->stack_counts[3] = total;
  const bool ok = S->n_sub[0] > 10 && S->n_sub[1] > 50;
  if (!ok) S->flags |= ALOAM_FLAG_MAP_TOO_THIN;
  S->stack_counts[2] = ok ? total : 0;   // zero residual blocks: the solve leaves the pose untouched, like the skipped optimisation
}
__global__ void k_mapper_prep(const __grid_constant__ Batch<MapperLane> B) { mapper_prep_body(B.a[blockIdx.z].S); }   // grid (1, 1, lanes)


// transformUpdate (:148-152): T_wmap_wodom from the map pose x (7 doubles: the frame's S->x, or an adopted recovery candidate)
// and the frame's odometry pose
__device__ __forceinline__ void transform_update(MapperState* S, const double* x) {
  const Qd qw{x[0], x[1], x[2], x[3]};
  const Qd qo{S->q_wodom[0], S->q_wodom[1], S->q_wodom[2], S->q_wodom[3]};
  const Qd qn = qmul(qw, qinv(qo));
  double r[3]; qrot(qn, S->t_wodom, r);
  S->q_wmap_wodom[0] = qn.x; S->q_wmap_wodom[1] = qn.y; S->q_wmap_wodom[2] = qn.z; S->q_wmap_wodom[3] = qn.w;
  S->t_wmap_wodom[0] = x[4] - r[0]; S->t_wmap_wodom[1] = x[5] - r[1]; S->t_wmap_wodom[2] = x[6] - r[2];
}
// transformUpdate ; refined pose out
__device__ __forceinline__ void mapper_update_body(MapperState* S, double* __restrict__ out7) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x || blockIdx.x) return;
  transform_update(S, S->x);
  if (out7) for (int k = 0; k < 7; ++k) out7[k] = S->x[k];
  S->frames++;
}
__global__ void k_mapper_update(const __grid_constant__ Batch<MapperLane> B) {   // grid (1, 1, lanes)
  const MapperLane& a = B.a[blockIdx.z];
  mapper_update_body(a.S, a.out7);
}


// end of the frame, after insertion and re-filter have set their error bits: a full cube, no free run, submap truncation and
// cubes left out of the re-filter become this frame's ALOAM_FLAG_CUBE_OVERFLOW, the frame's word joins the per-call accumulation, and `err` starts
// the next frame clear (everything of the next frame -- the stack filter forked onto the auxiliary stream included -- is
// ordered after this kernel)
__device__ __forceinline__ void mapper_finish_body(MapperState* S) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x || blockIdx.x) return;
  const int e = S->err;
  if (e & 30) S->flags |= ALOAM_FLAG_CUBE_OVERFLOW;
  S->frame_err = e;
  S->err_acc |= e;
  S->err = 0;
}
__global__ void k_mapper_finish(const __grid_constant__ Batch<MapperLane> B) { mapper_finish_body(B.a[blockIdx.z].S); }   // grid (1, 1, lanes)


// pointAssociateToMap (:154-163), then the cube of the stored point (:741-758)
// blockIdx.y = cloud (0 corner stack, 1 surf stack); the scratch of cloud 1 starts `scratch_stride` elements in
__device__ __forceinline__ void cube_ids_body(const Pt4* __restrict__ stack0, const Pt4* __restrict__ stack1, const MapperState* __restrict__ S, Pt4* __restrict__ world,
                           int* __restrict__ cube, int scratch_stride) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int which = blockIdx.y;
  const Pt4* __restrict__ stack = which ? stack1 : stack0;
  world += (size_t)which * scratch_stride; cube += (size_t)which * scratch_stride;
  const int n = S->stack_counts[which];
  const double ux = S->x[0], uy = S->x[1], uz = S->x[2], w = S->x[3], tx = S->x[4], ty = S->x[5], tz = S->x[6];
  const int c0 = S->cen[0], c1 = S->cen[1], c2 = S->cen[2];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const Pt4 s = point_associate_to_map(stack[i], ux, uy, uz, w, tx, ty, tz);
    const int ci = cube_coord((double)s.x, c0), cj = cube_coord((double)s.y, c1), ck = cube_coord((double)s.z, c2);
    world[i] = s;
    cube[i] = (ci >= 0 && ci < CW && cj >= 0 && cj < CH && ck >= 0 && ck < CD) ? cube_index(ci, cj, ck) : -1;
  }
}
// grid (CTAs, 2 clouds, lanes)
__global__ void k_cube_ids(const __grid_constant__ Batch<MapperLane> B, int scratch_stride) {
  const MapperLane& a = B.a[blockIdx.z];
  cube_ids_body(a.stack[0], a.stack[1], a.S, a.world, a.cube, scratch_stride);
}


// ---- the clouds the reference mapper publishes (:806-848)

// grid (points, 1, lanes): /velodyne_cloud_registered (:838-848) of a mapped scan -- its ring-major full-resolution cloud moved
// into the world frame by the frame's refined pose (pointAssociateToMap), read from S->x before the lane's next frame overwrites it
struct RegFullLane {
  const MapperState* S;
  const Pt4* src;   // the scan's ring-major cloud
  const int* n;     // its size (device)
  Pt4* dst;
};
__global__ void k_register_full(const __grid_constant__ Batch<RegFullLane> B) {
  const RegFullLane a = B.a[blockIdx.z];
  const MapperState* __restrict__ S = a.S;
  const double ux = S->x[0], uy = S->x[1], uz = S->x[2], w = S->x[3], tx = S->x[4], ty = S->x[5], tz = S->x[6];
  const int n = *a.n;
  const Pt4* __restrict__ src = a.src;
  Pt4* __restrict__ dst = a.dst;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = point_associate_to_map(src[i], ux, uy, uz, w, tx, ty, tz);
}

// ---- the exports of a store (aloam_mapper_export, lane snapshots, the prior map): the reference's order, corner cube then surf
// cube of every cube -- ALOAM_EXPORT_SURROUND the valid cubes of the last frame in laserCloudSurroundInd order (:806-821, the same
// loop as the valid list), ALOAM_EXPORT_MAP i = 0 .. 4850 (:823-836).  An ExportLayout says where each segment is in the export
// and in the store; k_store_copy moves points between the two.
constexpr long long kExportStage = 4ll << 20;   // points of the staging buffer of host memory (64 MB)

// One CTA of 1024 threads: the exclusive prefix of every thread's v over the block; s[1023] holds the total afterwards
template <typename T> __device__ T block_scan_1024(T v, T* s) {
  const int tid = threadIdx.x;
  s[tid] = v;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const T u = tid >= d ? s[tid - d] : T(0);
    __syncthreads();
    s[tid] += u;
    __syncthreads();
  }
  return s[tid] - v;
}

// one CTA of 1024: the layout L of export `what` of the store (S, slab pools p0 / p1 of cap0 / cap1 points per slab)
__global__ void __launch_bounds__(1024) k_export_sizes(const MapperState* __restrict__ S, int what, Pt4* p0, Pt4* p1, int cap0, int cap1, ExportLayout* __restrict__ L) {
  __shared__ long long s_part[1024];
  const int tid = threadIdx.x, nseg = what == ALOAM_EXPORT_SURROUND ? 2 * S->n_valid : kExportSegs;
  const int per = (nseg + 1023) / 1024, b = tid * per, e = min(b + per, nseg);
  auto slab = [&](int s) { return S->slab_of[s & 1][what == ALOAM_EXPORT_SURROUND ? S->valid[s >> 1] : s >> 1]; };
  long long sum = 0;
  for (int s = b; s < e; ++s) { const int k = slab(s); sum += k < 0 ? 0 : S->cnt[s & 1][k]; }
  long long run = block_scan_1024(sum, s_part);
  for (int s = b; s < e; ++s) {
    const int k = slab(s);
    L->off[s] = run;
    L->base[s] = k < 0 ? nullptr : (s & 1 ? p1 + (size_t)k * cap1 : p0 + (size_t)k * cap0);
    run += k < 0 ? 0 : S->cnt[s & 1][k];
  }
  if (tid == 1023) { L->off[nseg] = run; L->nseg = nseg; L->total = run; }
}

// grid-stride over the segments of layout L: the points of the window [lo, hi) of the export between io[position - lo] and the
// store -- to_store: io -> store, else store -> io
__global__ void __launch_bounds__(256) k_store_copy(const ExportLayout* __restrict__ L, Pt4* __restrict__ io, long long lo, long long hi, int to_store) {
  const int nseg = L->nseg;
  for (int s = blockIdx.x; s < nseg; s += gridDim.x) {
    const long long o = L->off[s], b = max(o, lo), e = min(L->off[s + 1], hi);
    if (b >= e) continue;   // (a segment with points has a base)
    Pt4* __restrict__ p = L->base[s];
    for (long long q = b + threadIdx.x; q < e; q += blockDim.x) {
      if (to_store) p[q - o] = io[q - lo]; else io[q - lo] = p[q - o];
    }
  }
}

// ---- lane snapshots (aloam_lane_restore): the inverse of the ALOAM_EXPORT_MAP export; seeded STARTs (aloam_lane_map_on_prior)

// the order of the run a cube of n points needs at cap points per slab: 0 for n <= cap, else the k with 2^k the next power of two
// of ceil(n / cap)
__host__ __device__ inline int run_order(int n, int cap) {
  int o = 0;
  while (((long long)cap << o) < n) ++o;
  return o;
}

// One CTA of 1024: the store whose cube i holds count(ty, i) points of type ty (-1: no slab), with runs of up to 2^ord0 corner /
// 2^ord1 surf slabs (every count fits its type's largest run: the caller has checked).  State of a fresh trajectory first, then
// every cube with a count >= 0 takes the run its count needs (run_order), packed from slab 0 up: the runs by decreasing size,
// cubes of one size in cube order, so every run is aligned (a size class starts at the sum of the larger ones).  When every run
// is one slab this is slabs 0, 1, 2, ... in cube order.  The rest of the pool stays free.  L = the layout of the ALOAM_EXPORT_MAP
// export of the new store.  The caller sets the fields that outlive a frame.
template <typename Count>
__device__ __forceinline__ void store_import_body(MapperState* __restrict__ S, Count count, Pt4* p0, Pt4* p1, int cap0, int cap1, int ord0, int ord1,
                                                  ExportLayout* __restrict__ L) {
  __shared__ long long s_pts[1024];
  __shared__ int s_scan[1024];
  __shared__ int s_top[2];
  const int tid = threadIdx.x;
  const int cap[2] = {cap0, cap1};
  mapper_fresh_state(S, ord0, ord1);
  if (tid < 2) s_top[tid] = 0;
  const int per = (NCUBE + 1023) / 1024, b = tid * per, e = min(b + per, NCUBE);
  long long pts = 0;
  int top[2] = {0, 0};
  for (int i = b; i < e; ++i)
    for (int ty = 0; ty < 2; ++ty) {
      const int n = count(ty, i);
      pts += max(n, 0);
      if (n >= 0) top[ty] = max(top[ty], run_order(n, cap[ty]));
    }
  __syncthreads();
  atomicMax(&s_top[0], top[0]); atomicMax(&s_top[1], top[1]);
  // (the first barrier of the scan also orders mapper_fresh_state's writes and the atomics before the ones below)
  long long run = block_scan_1024(pts, s_pts);
  for (int ty = 0; ty < 2; ++ty) {
    int base = 0;   // slabs the larger size classes take
    for (int o = s_top[ty]; o >= 0; --o) {
      int k = 0;
      for (int i = b; i < e; ++i) { const int n = count(ty, i); k += n >= 0 && run_order(n, cap[ty]) == o; }
      int slab = base + (block_scan_1024(k, s_scan) << o);
      base += s_scan[1023] << o;
      __syncthreads();   // s_scan is read before the next class overwrites it
      for (int i = b; i < e; ++i) {
        const int n = count(ty, i);
        if (n < 0 || run_order(n, cap[ty]) != o) continue;
        S->slab_of[ty][i] = slab; S->cnt[ty][slab] = n; S->ord[ty][slab] = (unsigned char)o;
        slab += 1 << o;
      }
    }
    if (tid < kPoolWords) S->used[ty][tid] = base >= 32 * (tid + 1) ? ~0u : base <= 32 * tid ? 0u : (1u << (base - 32 * tid)) - 1u;
  }
  for (int i = b; i < e; ++i)
    for (int ty = 0; ty < 2; ++ty) {
      const int s = count(ty, i) >= 0 ? S->slab_of[ty][i] : -1;   // (this thread wrote it)
      L->off[2 * i + ty] = run;
      L->base[2 * i + ty] = s < 0 ? nullptr : ty ? p1 + (size_t)s * cap1 : p0 + (size_t)s * cap0;
      if (s >= 0) run += S->cnt[ty][s];
    }
  if (tid == 1023) { L->off[kExportSegs] = run; L->nseg = kExportSegs; L->total = run; }
}

// the store a snapshot's table H describes (the caller has zeroed S), and the fields of H that outlive a frame
__global__ void __launch_bounds__(1024) k_store_import_tables(MapperState* __restrict__ S, const SnapStore* __restrict__ H, Pt4* p0, Pt4* p1, int cap0, int cap1,
                                                              int ord0, int ord1, ExportLayout* __restrict__ L) {
  store_import_body(S, [H](int ty, int i) { return H->count[ty][i]; }, p0, p1, cap0, cap1, ord0, ord1, L);
  const int tid = threadIdx.x;
  if (tid < kMaxValid) S->valid[tid] = tid < H->n_valid ? H->valid[tid] : 0;
  if (tid == 0) {
    for (int a = 0; a < 3; ++a) S->cen[a] = H->cen[a];
    S->n_valid = H->n_valid;
    S->frames = H->frames;
    for (int k = 0; k < 4; ++k) S->q_wmap_wodom[k] = H->q_wmap_wodom[k];
    for (int k = 0; k < 3; ++k) S->t_wmap_wodom[k] = H->t_wmap_wodom[k];
  }
}

// one seeded START: the lane's store, its slab pools and the layout its copy of the prior map gets, and the T_wmap_wodom it
// starts from (normalised by aloam_lane_map_on_prior)
struct SeedLane {
  MapperState* S;
  Pt4* pts[2];
  int cap[2];
  ExportLayout* L;
  double init[7];
};
// grid (1, 1, records), 1024 threads: record z's store becomes the prior map's (cube table cs [2][NCUBE + 1], centre offsets cen):
// every cube that holds points gets a run of its type as store_import_body packs them (one slab each with growth off: slabs 0,
// 1, 2, ... in cube order), the others none; runs of up to 2^ord0 / 2^ord1 slabs; frames = 0, an empty valid list and
// T_wmap_wodom = init.  Fields the stack filter writes (stack_counts, err, in_counts) stay as mapper_fresh_state leaves them.
__global__ void __launch_bounds__(1024) k_store_seed_tables(const __grid_constant__ Batch<SeedLane> B, const int* __restrict__ cs, int cen0, int cen1, int cen2,
                                                            int ord0, int ord1) {
  const SeedLane& a = B.a[blockIdx.z];
  MapperState* S = a.S;
  store_import_body(S, [cs](int ty, int i) { const int* t = cs + ty * (NCUBE + 1) + i; const int n = t[1] - t[0]; return n > 0 ? n : -1; },
                    a.pts[0], a.pts[1], a.cap[0], a.cap[1], ord0, ord1, a.L);
  if (threadIdx.x == 0) {
    S->cen[0] = cen0; S->cen[1] = cen1; S->cen[2] = cen2;
    for (int k = 0; k < 4; ++k) S->q_wmap_wodom[k] = a.init[k];
    for (int k = 0; k < 3; ++k) S->t_wmap_wodom[k] = a.init[4 + k];
  }
}

// grid-stride over the segments, grid (CTAs, 1, records): the points of record z's store (layout D[z]) from the prior map's (layout
// P).  Segment s of both layouts is the same cube and type with the same number of points.
__global__ void __launch_bounds__(256) k_store_seed_copy(const ExportLayout* __restrict__ P, const ExportLayout* __restrict__ D) {
  const ExportLayout* __restrict__ L = D + blockIdx.z;
  for (int s = blockIdx.x; s < kExportSegs; s += gridDim.x) {
    const int n = (int)(L->off[s + 1] - L->off[s]);
    if (n <= 0) continue;
    const Pt4* __restrict__ src = P->base[s];
    Pt4* __restrict__ dst = L->base[s];
    for (int q = threadIdx.x; q < n; q += blockDim.x) dst[q] = src[q];
  }
}


// The run of 2^o slabs at the lowest aligned free position of the occupancy bitmap whose word `lane` this warp lane holds in w
// (all 32 lanes call it with the same o): its first slab, marked used in w, or -1 when no aligned free run of that size exists.
__device__ __forceinline__ int take_run(unsigned& w, int o, int lane) {
  if (o <= 5) {   // the run lies inside one word
    const int n = 1 << o;
    unsigned g = ~w;
    for (int k = 1; k < n; k <<= 1) g &= g >> k;   // bit p: slabs p .. p + n - 1 of the word are free
    g &= (unsigned)(0xffffffffull / ((1ull << n) - 1ull));   // the aligned positions: every n-th bit from bit 0
    const unsigned hit = __ballot_sync(0xffffffffu, g != 0u);
    if (!hit) return -1;
    const int L = __ffs(hit) - 1, bit = __ffs(__shfl_sync(0xffffffffu, g, L)) - 1;
    if (lane == L) w |= run_mask(32 * L + bit, o, L);
    return 32 * L + bit;
  }
  const int q = 1 << (o - 5);   // whole words
  const unsigned m = q == 32 ? 0xffffffffu : (1u << q) - 1u;
  const unsigned empty = __ballot_sync(0xffffffffu, w == 0u);
  const unsigned hit = __ballot_sync(0xffffffffu, lane % q == 0 && ((empty >> lane) & m) == m);
  if (!hit) return -1;
  const int L = __ffs(hit) - 1;
  if (lane >= L && lane < L + q) w = 0xffffffffu;
  return 32 * L;
}

// stable append of the stack points to their cubes (push_back order = stack order, :759-767).  ONE CTA per cloud (blockIdx.x: the
// corner and the surf store are independent, the two appends run side by side), in four phases:
//   1. count: the points every cube gets and its first stack point;
//   2. runs: a cube that gets points and has no run, or whose run cannot hold its new count while a larger one is allowed, needs
//      the smallest run that holds min(new count, its ceiling) -- served by warp 0 in the order of the cubes' first stack points,
//      each from the lowest aligned free block of the bitmap; a cube whose run cannot be found keeps what it had (flagged);
//   3. move: a grown cube's points go to the start of its new run, in order; the old runs are freed once all are served;
//   4. append: the stack is walked in chunks of 1024; inside a chunk the warps take turns, the lanes of one cube form a group
//      (__match_any) whose leader advances the cube's running end in shared memory; a point beyond its cube's run is dropped.
// With growth off (max_ord 0) every run is one slab and no cube ever grows.  Dynamic shared memory: kInsertSmem bytes.
constexpr int kInsertSmem = 5 * NCUBE * (int)sizeof(int);
__device__ __forceinline__ void cube_insert_body(const Pt4* __restrict__ world, const int* __restrict__ cube, int scratch_stride, MapperState* S,
                                                      Pt4* __restrict__ pts0, int cap0, Pt4* __restrict__ pts1, int cap1) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int ty = blockIdx.x;
  world += (size_t)ty * scratch_stride; cube += (size_t)ty * scratch_stride;
  Pt4* __restrict__ pts = ty ? pts1 : pts0;
  const int cap = ty ? cap1 : cap0;
  extern __shared__ int s_dyn[];
  int* s_end = s_dyn;               // running end of every cube: its count before the insert, then the append's cursor
  int* s_slab = s_dyn + NCUBE;      // cube -> first slab of its run (the warps' turns must not wait on global memory)
  int* s_lim = s_dyn + 2 * NCUBE;   // points the stack brings, then the capacity of the cube's run (INT_MAX: no point comes)
  int* s_first = s_dyn + 3 * NCUBE; // its first stack point while it needs a run (INT_MAX otherwise), then its old run (-1: none)
  int* s_list = s_dyn + 4 * NCUBE;  // the cubes that need a run, in the order of their first stack point
  __shared__ int s_wsum[32], s_nlist;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = S->stack_counts[ty], max_ord = S->max_ord[ty];
  const int ceiling = cap << max_ord;
  int* slab_of = S->slab_of[ty];
  int* cnt = S->cnt[ty];
  unsigned char* ord = S->ord[ty];
  for (int c = tid; c < NCUBE; c += blockDim.x) {
    const int s = slab_of[c];
    s_slab[c] = s; s_end[c] = s < 0 ? 0 : cnt[s]; s_lim[c] = 0; s_first[c] = INT_MAX;
  }
  __syncthreads();
  // ---- 1. count
  for (int i = tid; i < n; i += blockDim.x) {
    const int c = cube[i];
    if (c >= 0) { atomicAdd(&s_lim[c], 1); atomicMin(&s_first[c], i); }
  }
  __syncthreads();
  // ---- 2. runs
  int need = 0;
  for (int c = tid; c < NCUBE; c += blockDim.x) {
    if (s_lim[c] == 0) continue;
    const int s = s_slab[c], o = run_order(min(s_end[c] + s_lim[c], ceiling), cap);
    if (s >= 0 && o <= ord[s]) s_first[c] = INT_MAX;
    else need = 1;
  }
  if (__syncthreads_or(need)) {
    if (tid == 0) s_nlist = 0;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {   // the cubes that need a run, compacted in stack order
      const int i = base + tid;
      const int c = i < n ? cube[i] : -1;
      const bool f = c >= 0 && s_first[c] == i;
      const unsigned bal = __ballot_sync(0xffffffffu, f);
      if (lane == 0) s_wsum[warp] = __popc(bal);
      __syncthreads();
      int off = s_nlist;
      for (int v = 0; v < warp; ++v) off += s_wsum[v];
      if (f) s_list[off + __popc(bal & ((1u << lane) - 1u))] = c;
      __syncthreads();
      if (tid == 0) { int t = 0; for (int v = 0; v < 32; ++v) t += s_wsum[v]; s_nlist += t; }
      __syncthreads();
    }
    const int nl = s_nlist;
    if (warp == 0) {
      unsigned w = S->used[ty][lane];
      for (int k = 0; k < nl; ++k) {
        const int c = s_list[k], old = s_slab[c];
        const int o = run_order(min(s_end[c] + s_lim[c], ceiling), cap);
        const int s = take_run(w, o, lane);
        if (lane == 0) {
          s_first[c] = -1;
          if (s < 0) atomicOr(&S->err, 4);   // no free run of that size: the cube keeps what it had
          else { s_slab[c] = s; ord[s] = (unsigned char)o; s_first[c] = old; }
        }
      }
      __syncwarp();
      for (int k = 0; k < nl; ++k) {   // the old runs of grown cubes go back to the pool once every run is served
        const int old = s_first[s_list[k]];
        if (old >= 0) { const unsigned m = run_mask(old, ord[old], lane); w &= ~m; }
      }
      S->used[ty][lane] = w;
    }
    __syncthreads();
    // ---- 3. move
    for (int k = 0; k < nl; ++k) {
      const int c = s_list[k], old = s_first[c];
      if (old < 0) continue;
      const Pt4* __restrict__ src = pts + (size_t)old * cap;
      Pt4* __restrict__ dst = pts + (size_t)s_slab[c] * cap;
      for (int q = tid; q < s_end[c]; q += blockDim.x) dst[q] = src[q];
      if (tid == 0) cnt[old] = 0;
    }
  }
  for (int c = tid; c < NCUBE; c += blockDim.x) {
    const int s = s_slab[c];
    s_lim[c] = s_lim[c] == 0 ? INT_MAX : s < 0 ? 0 : cap << ord[s];
  }
  __syncthreads();
  // ---- 4. append
  for (int base = 0; base < n; base += 1024) {
    const int i = base + tid;
    const int mine = i < n ? cube[i] : -1;
    const Pt4 p = i < n ? world[i] : Pt4{0.f, 0.f, 0.f, 0.f};
    const int warps = min(32, (n - base + 31) / 32);
    for (int w = 0; w < warps; ++w) {
      if (warp == w) {
        const unsigned grp = __match_any_sync(0xffffffffu, mine);
        const int leader = __ffs(grp) - 1;
        int start = 0, slab = -1, lim = 0;
        if (mine >= 0 && lane == leader) {
          slab = s_slab[mine];
          lim = s_lim[mine];
          start = s_end[mine];
          s_end[mine] = start + __popc(grp);
        }
        start = __shfl_sync(0xffffffffu, start, leader);
        slab = __shfl_sync(0xffffffffu, slab, leader);
        lim = __shfl_sync(0xffffffffu, lim, leader);
        if (mine >= 0 && slab >= 0) {
          const int pos = start + __popc(grp & ((1u << lane) - 1u));
          if (pos < lim) pts[(size_t)slab * cap + pos] = p;
          else atomicOr(&S->err, 2);   // the cube's run is full: the overflow is dropped (flagged), the frame goes on
        }
      }
      __syncthreads();
    }
  }
  for (int c = tid; c < NCUBE; c += blockDim.x) { const int s = s_slab[c]; if (s >= 0) { slab_of[c] = s; cnt[s] = min(s_end[c], s_lim[c]); } }
}
// grid (2 clouds, 1, lanes), kInsertSmem bytes of dynamic shared memory: every CTA has its own shared cube tables and takes runs
// from its lane's pool
__global__ void __launch_bounds__(1024) k_cube_insert(const __grid_constant__ Batch<MapperLane> B, int scratch_stride) {
  const MapperLane& a = B.a[blockIdx.z];
  cube_insert_body(a.world, a.cube, scratch_stride, a.S, a.pts[0], a.cap[0], a.pts[1], a.cap[1]);
}


// segment descriptors of the per-cube re-filter (:770-801): the valid cubes, corner cubes then surf cubes, in place -- as long as
// their running total fits the filter's buffer of `budget` points.  The cubes from the first one that does not fit on are left
// unfiltered for this frame (flagged: err bit 4).  With growth off a cube holds at most one slab and every valid cube fits.
__device__ __forceinline__ void seg_cubes_body(MapperState* S, SegDesc* segs, int* n_seg, Pt4* p0, Pt4* p1, int cap0, int cap1, float leaf0, float leaf1,
                                               int budget) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  __shared__ int s_w[8];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5, nv = S->n_valid;
  int s = -1, n = 0;
  if (t < 2 * nv) {
    const int ty = t >= nv, v = ty ? t - nv : t;
    s = S->slab_of[ty][S->valid[v]];
    n = s < 0 ? 0 : S->cnt[ty][s];
  }
  // the running total through this cube (block scan; <= 150 x 2^18 points fits int): the counts are >= 0, so the cubes that fit
  // are a prefix of the list
  int incl = n;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
  if (lane == 31) s_w[w] = incl;
  __syncthreads();
  for (int v = 0; v < w; ++v) incl += s_w[v];
  const int keep = __syncthreads_count(t < 2 * nv && incl <= budget);
  if (t == 0) {
    if (keep < 2 * nv) atomicOr(&S->err, 16);
    *n_seg = keep; S->zero = 0;
  }
  if (t < keep) {
    const int ty = t >= nv;
    Pt4* base = s < 0 ? (ty ? p1 : p0) : (ty ? p1 : p0) + (size_t)s * (ty ? cap1 : cap0);
    int* np = s < 0 ? &S->zero : &S->cnt[ty][s];
    segs[t] = SegDesc{base, np, ty ? leaf1 : leaf0, base, s < 0 ? &S->sink : np};
  }
}
// grid (1, 1, lanes)
__global__ void __launch_bounds__(256) k_seg_cubes(const __grid_constant__ Batch<MapperLane> B, float leaf0, float leaf1, int budget) {
  const MapperLane& a = B.a[blockIdx.z];
  seg_cubes_body(a.S, a.segs, a.n_seg, a.pts[0], a.pts[1], a.cap[0], a.cap[1], leaf0, leaf1, budget);
}


// points one segmented filter can sort: the re-filter takes every point of the <= 75 valid cubes of each type, full slabs
// included (the submap gather truncates only its own copy at max_map_points), the stack filter two scan clouds
size_t refilter_bound(const Mapper* m, const aloam_ctx* c) {
  return std::max((size_t)75 * (m->cap[0] + m->cap[1]), (size_t)2 * c->max_points);
}

// the state of a fresh trajectory (mapper_fresh_state, the routine k_mapper_begin runs for a lane that starts one), with the
// fields that routine leaves alone zeroed first, under the context's cube growth
int reset_lane(aloam_ctx* c, Mapper* m) {
  int ord[2];
  mapper_run_orders(c, c->cube_growth, ord);
  CUDA_CHECK_RET(cudaMemsetAsync(m->frame.d_state, 0, sizeof(MapperState), c->stream));
  LAUNCH(c, KID_CUBES, k_mapper_reset, 1, 1024, 0, m->frame.d_state, ord[0], ord[1]);
  CUDA_CHECK_RET(cudaGetLastError());
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  return ALOAM_OK;
}

// the stream and events of the stack filters' fork (stack_filters_fork), created with the first cube store or locator
cudaError_t stack_stream_ensure(aloam_ctx* c) {
  if (c->ev_stack_join) return cudaSuccess;
  cudaError_t e = screate(c, &c->s_stack);
  if (e == cudaSuccess) e = ecreate(c, &c->ev_stack_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = ecreate(c, &c->ev_stack_join, cudaEventDisableTiming);
  return e;
}

// the two scan-stack filters of a frame (:541-550) as one segmented pass over both clouds of every lane (records B, filters f on
// buffers bufs), on s_stack: they read only the scans' clouds, so they run beside what the frame issues next on c->stream until
// the caller joins on ev_stack_join
int stack_filters_fork(aloam_ctx* c, int nb, const Batch<MapperLane>& B, const SegFilter* f, SegBuffers* const* bufs, int n_upper_c, int n_upper_s) {
  cudaStream_t main_stream = c->stream;
  CUDA_CHECK_RET(cudaEventRecord(c->ev_stack_fork, main_stream));
  CUDA_CHECK_RET(cudaStreamWaitEvent(c->s_stack, c->ev_stack_fork, 0));
  c->stream = c->s_stack;
  launch_ex(c, KID_VOXEL, k_seg_two, dim3(1, 1, nb), dim3(32), 0, 1, false, B, c->cfg.line_res, c->cfg.plane_res);
  vox_seg_filter(c, nb, f, bufs, 2, n_upper_c + n_upper_s, std::max(n_upper_c, n_upper_s));
  const cudaError_t e = cudaEventRecord(c->ev_stack_join, c->s_stack);
  c->stream = main_stream;
  CUDA_CHECK_RET(e);
  return ALOAM_OK;
}

// the layout of export `what` of the store of m into c->d_export_layout (created on first use); *n = the size of the export.
// Synchronises.
int export_sizes(aloam_ctx* c, const Mapper* m, int what, long long* n) {
  if (!c->d_export_layout) CUDA_CHECK_RET(dalloc(c, &c->d_export_layout, 1));
  LAUNCH(c, KID_CUBES, k_export_sizes, 1, 1024, 0, m->frame.d_state, what, m->d_pts[0], m->d_pts[1], m->cap[0], m->cap[1], c->d_export_layout);
  CUDA_CHECK_RET(cudaMemcpyAsync(&c->pin->export_total, &c->d_export_layout->total, sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  *n = c->pin->export_total;
  return ALOAM_OK;
}

// the points [0, n) of the export layout L describes, between the store and `mem` (to_store: mem -> store, else store -> mem), on
// c->stream, not synchronised: device memory in place, host memory through the staging buffer (created on first use) one window
// at a time, copied in before the window's launch or out after it
int store_copy(aloam_ctx* c, const ExportLayout* L, long long n, char* mem, bool device, bool to_store) {
  const int blocks = std::min(kExportSegs, c->sms * 8);
  if (device) {
    LAUNCH(c, KID_CUBES, k_store_copy, blocks, 256, 0, L, reinterpret_cast<Pt4*>(mem), 0ll, n, (int)to_store);
  } else {
    if (!c->d_export_stage) CUDA_CHECK_RET(dalloc(c, &c->d_export_stage, (size_t)kExportStage));
    for (long long lo = 0; lo < n; lo += kExportStage) {
      const long long hi = std::min(n, lo + kExportStage);
      const size_t bytes = (size_t)(hi - lo) * sizeof(Pt4);
      if (to_store) CUDA_CHECK_RET(cudaMemcpyAsync(c->d_export_stage, mem + lo * sizeof(Pt4), bytes, cudaMemcpyHostToDevice, c->stream));
      LAUNCH(c, KID_CUBES, k_store_copy, blocks, 256, 0, L, c->d_export_stage, lo, hi, (int)to_store);
      if (!to_store) CUDA_CHECK_RET(cudaMemcpyAsync(mem + lo * sizeof(Pt4), c->d_export_stage, bytes, cudaMemcpyDeviceToHost, c->stream));
    }
  }
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}


// ---- localisation: the prior map of a context and the lanes that register against it

// the one place a context's prior map is released: aloam_prior_map_clear, a load that replaces it, aloam_destroy
void prior_map_release(aloam_ctx* c) {
  delete c->prior;
  c->prior = nullptr;
  for (Lane& L : c->lanes) L.window = false;   // the windows were cut from this map
}

// The record of frame f for `in` with the fields every frame fills -- state, poses, input clouds and sizes, stacks, segment
// descriptors -- and the stack filter of f into *stack_f / *buf; a mapping frame adds its store's fields
MapperLane frame_record(LaneFrame* f, const MapperIn& in, SegFilter* stack_f, SegBuffers** buf) {
  MapperState* S = f->d_state;
  *stack_f = seg_filter(f->buf, 31, &S->err);
  *buf = &f->buf;
  MapperLane a = {};
  a.S = S; a.odom7 = in.odom7; a.out7 = in.out7;
  a.in[0] = in.corner; a.in[1] = in.surf; a.n_in[0] = in.nc; a.n_in[1] = in.ns;
  a.stack[0] = f->reg->stack[0]; a.stack[1] = f->reg->stack[1];
  a.segs = f->buf.segs; a.n_seg = f->buf.n_seg;
  return a;
}

// the persistent index: the k_grid_* chain of mapping.cu once over both packed clouds, then the cube tags
void prior_index(aloam_ctx* c, PriorMap* p) {
  Batch<GridArgs> g = {};
  g.a[0] = GridArgs{p->grid[0], p->pts[0], p->d_n, p->grid[1], p->pts[1], p->d_n + 1};
  const int n_upper = std::max(1, std::max(p->n[0], p->n[1]));
  const int wave = c->sms * 8;
  const int pb = std::min((n_upper + 255) / 256, wave);
  const int tb = std::min((int)((std::max(p->grid[0].cap_slots, p->grid[1].cap_slots) + 255) / 256), wave);
  LAUNCH(c, KID_MAP_GRID, k_grid_setup, 1, 32, 0, g);
  LAUNCH(c, KID_MAP_GRID, k_grid_clear, dim3(tb, 1, 1), 256, 0, g);
  LAUNCH(c, KID_MAP_GRID, k_grid_insert, dim3(pb, 2, 1), 256, 0, g, 0, 1);
  LAUNCH(c, KID_MAP_GRID, k_grid_alloc, dim3(tb, 1, 1), 256, 0, g);
  LAUNCH(c, KID_MAP_GRID, k_grid_fill, dim3(pb, 2, 1), 256, 0, g);
  LAUNCH(c, KID_MAP_GRID, k_prior_tag, dim3(pb, 2, 1), 256, 0, p->grid[0], p->grid[1], p->d_cube_start);
}

// Makes a new map the context's prior map: centre offsets cen, cloud t of cs[t][NCUBE] points with cube i at [cs[t][i], cs[t][i + 1])
// (cs in host memory, 2 x (NCUBE + 1) ints).  Allocates the map, uploads the cube table and the ALOAM_EXPORT_MAP layout, lets
// fill(p) write the points of p->pts[0 / 1] on c->stream (returns an ALOAM_* code), builds the index, synchronises and swaps the
// map in.  The old map is replaced only on success; on failure the new one is freed.  aloam_prior_map_load and
// aloam_prior_map_build end here.
template <typename Fill> int prior_install(aloam_ctx* c, const int cen[3], const std::vector<int>& cs, Fill fill) {
  PriorMap* p = new (std::nothrow) PriorMap();
  if (!p) return ALOAM_ERR_CUDA;
  int cap[2];
  mapper_slab_caps(c, cap);
  for (int t = 0; t < 2; ++t) {
    p->n[t] = cs[(size_t)t * (NCUBE + 1) + NCUBE];
    for (int i = 0; i < NCUBE; ++i) {
      const int n = cs[(size_t)t * (NCUBE + 1) + i + 1] - cs[(size_t)t * (NCUBE + 1) + i];
      p->max_cube[t] = std::max(p->max_cube[t], n);
      p->n_cubes[t] += n > 0;
      if (n > 0) p->run_slabs[t] = (int)std::min<long long>((long long)p->run_slabs[t] + (1ll << std::min(run_order(n, cap[t]), 30)), INT_MAX);
    }
  }
  for (int a = 0; a < 3; ++a) p->cen[a] = cen[a];
  bool ok = p->mem.dev(&p->d_cube_start, cs.size()) && p->mem.dev(&p->d_n, 2) && p->mem.dev(&p->d_layout, 1);
  for (int t = 0; t < 2 && ok; ++t) {
    GridTable& g = p->grid[t];
    g.cap_slots = grid_mask_for(p->n[t], 1u << 30) + 1;
    g.cs = kMapCell; g.inv_cs = 1.0f / g.cs;
    const size_t n1 = (size_t)std::max(p->n[t], 1);
    ok = p->mem.dev(&p->pts[t], n1) && p->mem.dev(&g.gpts, n1) && p->mem.dev(&g.slots, (size_t)g.cap_slots) && p->mem.dev(&g.dyn, 1);
  }
  auto fail = [&](int code) { cudaStreamSynchronize(c->stream); cudaGetLastError(); delete p; return code; };
  if (!ok) return fail(ALOAM_ERR_CUDA);
  // the ALOAM_EXPORT_MAP layout of the packed clouds: segment 2 i + t is cube i of cloud t
  std::unique_ptr<ExportLayout> L(new (std::nothrow) ExportLayout());
  if (!L) return fail(ALOAM_ERR_CUDA);
  L->nseg = kExportSegs;
  for (int s = 0; s < kExportSegs; ++s) {
    const int* t = &cs[(size_t)(s & 1) * (NCUBE + 1) + (s >> 1)];
    L->base[s] = p->pts[s & 1] + t[0];
    L->off[s + 1] = L->off[s] + (t[1] - t[0]);
  }
  L->total = L->off[kExportSegs];
  if (cudaMemcpyAsync(p->d_cube_start, cs.data(), cs.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
      cudaMemcpyAsync(p->d_n, p->n, 2 * sizeof(int), cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
      cudaMemcpyAsync(p->d_layout, L.get(), sizeof(ExportLayout), cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
    return fail(ALOAM_ERR_CUDA);
  const int rc = fill(p); if (rc) return fail(rc);
  prior_index(c, p);
  if (cudaStreamSynchronize(c->stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) return fail(ALOAM_ERR_CUDA);
  if (!c->prior_owned) { own(c, [c] { prior_map_release(c); }); c->prior_owned = true; }
  prior_map_release(c);
  c->prior = p;
  for (Lane& L : c->lanes) if (L.sched.arm == ARM_MAP_ON_PRIOR) L.sched.arm = ARM_NONE;   // its fit was checked against the old map
  return ALOAM_OK;
}

// ---- building a prior map from two map-frame clouds (aloam_prior_map_build): the insertion of laserMapping.cpp:741-767 for every
// point at once, then the per-cube VoxelGrid of :787-801 over every cube.  Segment s = t NCUBE + i holds the points of type t in
// cube i; kBuildSegs marks a dropped point.  Order of launches: k_build_init, k_build_classify (cube, finite check, per-segment
// counts and boxes), k_build_params (min_b / div_b / PCL's overflow test per segment, segment offsets), k_build_keys (voxel index
// of every point), two stable sorts (voxel index, then segment: lexicographic), k_build_heads / k_build_scan (run starts and their
// ranks), k_build_ranks (voxels before every segment) -- one synchronisation to learn the map's sizes -- then k_build_emit writes
// every voxel's centroid straight into the map at its rank.
constexpr int kBuildSegs = 2 * NCUBE;
constexpr int kBuildTile = 256;

struct BuildSeg {
  int min_b[3], div_b[3];
  float inv;
  int pass;   // PCL's "leaf size is too small": the cube's points are kept as they are, in input order
};

// one coordinate's cube index (laserMapping.cpp:741-750), decided in double before any conversion: false when (v + 25) / 50 is
// not finite or lies beyond int, which the reference leaves undefined (the conversion is undefined on the CPU, saturates on the GPU)
__device__ __forceinline__ bool build_cube_coord(float v, int centre, long long* out) {
  const double s = (double)v + 25.0;
  const double q = s / 50.0;
  if (!(q > -2147483649.0 && q < 2147483648.0)) return false;
  *out = (long long)(int)q + centre - (s < 0 ? 1 : 0);
  return true;
}

__device__ __forceinline__ int build_f2ord(float f) { const int i = __float_as_int(f); return i >= 0 ? i : (i ^ 0x7fffffff); }
__device__ __forceinline__ float build_ord2f(int i) { return __int_as_float(i >= 0 ? i : (i ^ 0x7fffffff)); }

__global__ void __launch_bounds__(256) k_build_init(int* __restrict__ cnt, int* __restrict__ bbox, int* __restrict__ dropped) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < kBuildSegs) {
    cnt[s] = 0;
    for (int a = 0; a < 3; ++a) { bbox[6 * s + a] = INT_MAX; bbox[6 * s + 3 + a] = INT_MIN; }
  }
  if (s < 2) dropped[s] = 0;
}

// grid-stride over the n points (corner [0, n_c), surf after): seg[i], and per segment the count and the bounding box (atomics on
// the order-preserving int of the float, once per group of a warp's lanes that share a segment); dropped[t] per type
__global__ void __launch_bounds__(256) k_build_classify(const Pt4* __restrict__ pts, int n_c, int n, int c0, int c1, int c2, int* __restrict__ seg,
                                                        int* __restrict__ cnt, int* __restrict__ bbox, int* __restrict__ dropped) {
  const int lane = threadIdx.x & 31;
  for (int base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const int i = base + threadIdx.x;
    int s = -1;   // -1: no point; kBuildSegs + t: a dropped point of type t
    Pt4 p = {0.f, 0.f, 0.f, 0.f};
    if (i < n) {
      p = pts[i];
      long long a = -1, b = -1, d = -1;
      const bool ok = build_cube_coord(p.x, c0, &a) && build_cube_coord(p.y, c1, &b) && build_cube_coord(p.z, c2, &d) &&
                      a >= 0 && a < CW && b >= 0 && b < CH && d >= 0 && d < CD;   // :751-756
      const int t = i >= n_c ? 1 : 0;
      s = ok ? t * NCUBE + (int)(a + CW * b + CW * CH * d) : kBuildSegs + t;
      seg[i] = ok ? s : kBuildSegs;
    }
    const unsigned grp = __match_any_sync(0xffffffffu, s);
    const bool leader = lane == __ffs(grp) - 1;
    if (s >= kBuildSegs) {
      if (leader) atomicAdd(&dropped[s - kBuildSegs], __popc(grp));
    } else if (s >= 0) {
      const int lo[3] = {__reduce_min_sync(grp, build_f2ord(p.x)), __reduce_min_sync(grp, build_f2ord(p.y)), __reduce_min_sync(grp, build_f2ord(p.z))};
      const int hi[3] = {__reduce_max_sync(grp, build_f2ord(p.x)), __reduce_max_sync(grp, build_f2ord(p.y)), __reduce_max_sync(grp, build_f2ord(p.z))};
      if (leader) {
        atomicAdd(&cnt[s], __popc(grp));
        for (int k = 0; k < 3; ++k) { atomicMin(&bbox[6 * s + k], lo[k]); atomicMax(&bbox[6 * s + 3 + k], hi[k]); }
      }
    }
  }
}

// one CTA of 1024: every segment's voxel parameters, as seg_keys_body (voxel.cu) derives them from the segment's box; off = the
// exclusive prefix of the counts (off[kBuildSegs] = the points kept)
__global__ void __launch_bounds__(1024) k_build_params(const int* __restrict__ cnt, const int* __restrict__ bbox, float leaf0, float leaf1,
                                                       BuildSeg* __restrict__ par, int* __restrict__ off) {
  __shared__ int s_part[1024];
  const int per = (kBuildSegs + 1023) / 1024, b = threadIdx.x * per, e = min(b + per, kBuildSegs);
  int sum = 0;
  for (int s = b; s < e; ++s) sum += cnt[s];
  int run = block_scan_1024(sum, s_part);
  for (int s = b; s < e; ++s) {
    off[s] = run;
    run += cnt[s];
    BuildSeg g = {};
    if (cnt[s] > 0) {
      const float inv = 1.0f / (s < NCUBE ? leaf0 : leaf1);
      long long dxyz[3];
      for (int a = 0; a < 3; ++a) {
        const float mn = build_ord2f(bbox[6 * s + a]), mx = build_ord2f(bbox[6 * s + 3 + a]);
        dxyz[a] = (long long)((mx - mn) * inv) + 1;
        g.min_b[a] = (int)floorf(mn * inv);
        g.div_b[a] = (int)floorf(mx * inv) - g.min_b[a] + 1;
      }
      g.inv = inv;
      // PCL's test in int64 (dx dy dz > INT_MAX); in double here so that no product overflows -- exact while it matters
      g.pass = (double)dxyz[0] * (double)dxyz[1] * (double)dxyz[2] > (double)INT_MAX;
    }
    par[s] = g;
  }
  if (threadIdx.x == 1023) off[kBuildSegs] = run;
}

// grid-stride: vox[i] = PCL's voxel index of point i in its segment's box (0 in a pass-through segment and for a dropped point,
// whose order the stable sorts keep); keys / values of the first sort
__global__ void __launch_bounds__(256) k_build_keys(const Pt4* __restrict__ pts, int n, const int* __restrict__ seg, const BuildSeg* __restrict__ par,
                                                    unsigned* __restrict__ vox, unsigned* __restrict__ keys, int* __restrict__ vals) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int s = seg[i];
    unsigned idx = 0;
    if (s < kBuildSegs && !par[s].pass) {
      const BuildSeg& g = par[s];
      const Pt4 p = pts[i];
      const int i0 = (int)(floorf(p.x * g.inv) - (float)g.min_b[0]);
      const int i1 = (int)(floorf(p.y * g.inv) - (float)g.min_b[1]);
      const int i2 = (int)(floorf(p.z * g.inv) - (float)g.min_b[2]);
      idx = (unsigned)i0 + (unsigned)i1 * (unsigned)g.div_b[0] + (unsigned)i2 * ((unsigned)g.div_b[0] * (unsigned)g.div_b[1]);   // PCL's int, wrapped
    }
    vox[i] = idx;
    keys[i] = idx;
    vals[i] = i;
  }
}

// grid-stride: the keys of the second sort, the segment of the point at every slot of the first
__global__ void __launch_bounds__(256) k_build_gather(const int* __restrict__ seg, int n, unsigned* __restrict__ keys, const int* __restrict__ vals) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) keys[j] = (unsigned)seg[vals[j]];
}

// one thread per sorted slot, a tile of kBuildTile per CTA: head[j] = slot j starts a voxel (every slot of a pass-through segment
// does; a dropped point never does); tile_heads = heads per tile
__global__ void __launch_bounds__(kBuildTile) k_build_heads(const unsigned* __restrict__ sseg, const int* __restrict__ sval, int n, const unsigned* __restrict__ vox,
                                                            const BuildSeg* __restrict__ par, unsigned char* __restrict__ head, int* __restrict__ tile_heads) {
  const int j = blockIdx.x * kBuildTile + threadIdx.x;
  bool h = false;
  if (j < n) {
    const unsigned s = sseg[j];
    h = s < (unsigned)kBuildSegs && (j == 0 || s != sseg[j - 1] || par[s].pass || vox[sval[j]] != vox[sval[j - 1]]);
    head[j] = h ? 1 : 0;
  }
  const int cnt = __syncthreads_count(h);
  if (threadIdx.x == 0) tile_heads[blockIdx.x] = cnt;
}

// one CTA of 1024: exclusive scan of the tiles' head counts in place; *total = all heads
__global__ void __launch_bounds__(1024) k_build_scan(int* __restrict__ tile_heads, int tiles, int* __restrict__ total) {
  __shared__ int s_part[1024];
  const int per = (tiles + 1023) / 1024, b = threadIdx.x * per, e = min(b + per, tiles);
  int sum = 0;
  for (int k = b; k < e; ++k) sum += tile_heads[k];
  int run = block_scan_1024(sum, s_part);
  for (int k = b; k < e; ++k) { const int v = tile_heads[k]; tile_heads[k] = run; run += v; }
  if (threadIdx.x == 1023) *total = run;
}

// one warp per segment s <= kBuildSegs: rank[s] = voxels before the segment's first sorted slot off[s]
__global__ void __launch_bounds__(32) k_build_ranks(const int* __restrict__ off, const unsigned char* __restrict__ head, const int* __restrict__ tile_off,
                                                    const int* __restrict__ total, int n, int* __restrict__ rank) {
  const int s = blockIdx.x, pos = off[s];
  if (pos >= n) { if (threadIdx.x == 0) rank[s] = *total; return; }
  const int t = pos / kBuildTile;
  int c = 0;
  for (int j = t * kBuildTile + threadIdx.x; j < pos; j += 32) c += head[j];
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if (threadIdx.x == 0) rank[s] = tile_off[t] + c;
}

// one thread per sorted slot: a head sums its voxel's run in sorted order (float, pcl::CentroidPoint) and writes the centroid to
// its rank in the map (cloud 0 below n0 voxels, cloud 1 after); a pass-through head copies its point (keeps -0.f)
__global__ void __launch_bounds__(kBuildTile) k_build_emit(const Pt4* __restrict__ pts, const unsigned* __restrict__ sseg, const int* __restrict__ sval, int n,
                                                           const BuildSeg* __restrict__ par, const unsigned char* __restrict__ head,
                                                           const int* __restrict__ tile_off, int n0, Pt4* __restrict__ out0, Pt4* __restrict__ out1) {
  __shared__ int s_w[kBuildTile / 32];
  const int j = blockIdx.x * kBuildTile + threadIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const bool h = j < n && head[j];
  const unsigned bal = __ballot_sync(0xffffffffu, h);
  if (lane == 0) s_w[w] = __popc(bal);
  __syncthreads();
  if (!h) return;
  int r = tile_off[blockIdx.x] + __popc(bal & ((1u << lane) - 1u));
  for (int v = 0; v < w; ++v) r += s_w[v];
  const unsigned s = sseg[j];
  Pt4* dst = s < NCUBE ? out0 + r : out1 + (r - n0);
  if (par[s].pass) { *dst = pts[sval[j]]; return; }
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  int cnt = 0;
  for (int k = j; k < n && (k == j || (!head[k] && sseg[k] == s)); ++k) {
    const Pt4 p = pts[sval[k]];
    sx += p.x; sy += p.y; sz += p.z; si += p.i;
    ++cnt;
  }
  const float nf = (float)cnt;
  Pt4 o; o.x = sx / nf; o.y = sy / nf; o.z = sz / nf; o.i = si / nf;
  *dst = o;
}

// the build's scratch, one group: freed (after the stream has drained) when the call returns
struct BuildScratch {
  cudaStream_t stream;
  BufGroup mem;
  Pt4* pts = nullptr;
  int *seg = nullptr, *cnt = nullptr, *bbox = nullptr, *dropped = nullptr, *off = nullptr, *vals[2] = {nullptr, nullptr}, *hist = nullptr;
  int *tile_heads = nullptr, *total = nullptr, *rank = nullptr, *n_dev = nullptr;
  unsigned *vox = nullptr, *keys[2] = {nullptr, nullptr};
  unsigned char* head = nullptr;
  BuildSeg* par = nullptr;
  explicit BuildScratch(cudaStream_t s) : stream(s) {}
  ~BuildScratch() {   // runs before `mem` is freed
    cudaStreamSynchronize(stream);
    cudaGetLastError();
  }
  bool alloc(size_t n, int tiles) {
    const size_t n1 = std::max<size_t>(n, 1);
    return mem.dev(&pts, n1) && mem.dev(&seg, n1) && mem.dev(&cnt, kBuildSegs) && mem.dev(&bbox, 6 * kBuildSegs) && mem.dev(&dropped, 2) &&
           mem.dev(&off, kBuildSegs + 1) && mem.dev(&vals[0], n1) && mem.dev(&vals[1], n1) && mem.dev(&hist, vox_radix_hist_ints((int)n1)) &&
           mem.dev(&tile_heads, (size_t)std::max(tiles, 1)) && mem.dev(&total, 1) && mem.dev(&rank, kBuildSegs + 1) && mem.dev(&n_dev, 1) &&
           mem.dev(&vox, n1) && mem.dev(&keys[0], n1) && mem.dev(&keys[1], n1) && mem.dev(&head, n1) && mem.dev(&par, kBuildSegs);
  }
};

}  // namespace

// points per slab of the two cloud types (16 k corner / 64 k surf, at most cfg.max_points)
void mapper_slab_caps(const aloam_ctx* c, int cap[2]) {
  cap[0] = std::min(16384, c->max_points);
  cap[1] = std::min(65536, c->max_points);
}

// the largest run of a lane store per type, 2^ord[t] slabs: with growth on the largest power of two r with r x cap <=
// ALOAM_MAX_CUBE_POINTS (and r <= the pool), else one slab
void mapper_run_orders(const aloam_ctx* c, bool growth, int ord[2]) {
  int cap[2];
  mapper_slab_caps(c, cap);
  for (int t = 0; t < 2; ++t) {
    ord[t] = 0;
    while (growth && ord[t] < kMaxOrder && ((long long)cap[t] << (ord[t] + 1)) <= ALOAM_MAX_CUBE_POINTS) ++ord[t];
  }
}

// ---- lane snapshots (snapshot.cu): the cube store of a lane in the slab-free form of SnapStore

// the table of lane `lane`'s store into *head (host memory): the fields that outlive a frame and every cube's point count, -1 for a
// cube without a run; head->n_points = the size of the ALOAM_EXPORT_MAP export; *growth = the store's cube growth.  The store
// exists.  Synchronises.
int mapper_store_tables(aloam_ctx* c, int lane, SnapStore* head, int* growth) {
  Mapper* m = c->lanes[lane].mapper;
  CUDA_CHECK_RET(cudaMemcpyAsync(m->frame.h_state, m->frame.d_state, sizeof(MapperState), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  const MapperState* S = m->frame.h_state;
  std::memset(head, 0, sizeof(*head));
  for (int a = 0; a < 3; ++a) head->cen[a] = S->cen[a];
  head->n_valid = S->n_valid;
  for (int v = 0; v < S->n_valid; ++v) head->valid[v] = S->valid[v];
  head->frames = S->frames;
  for (int k = 0; k < 4; ++k) head->q_wmap_wodom[k] = S->q_wmap_wodom[k];
  for (int k = 0; k < 3; ++k) head->t_wmap_wodom[k] = S->t_wmap_wodom[k];
  long long n = 0;
  for (int ty = 0; ty < 2; ++ty)
    for (int i = 0; i < NCUBE; ++i) {
      const int s = S->slab_of[ty][i];
      head->count[ty][i] = s < 0 ? -1 : S->cnt[ty][s];
      n += s < 0 ? 0 : S->cnt[ty][s];
    }
  head->n_points = n;
  *growth = S->max_ord[0] > 0;
  return ALOAM_OK;
}

// the n points of lane `lane`'s store in ALOAM_EXPORT_MAP order into dst (device memory when `device`, else host memory), on
// c->stream, not synchronised; n is what mapper_store_tables reported (ALOAM_ERR_STATE when the store disagrees)
int mapper_store_points(aloam_ctx* c, int lane, long long n, char* dst, bool device) {
  const Mapper* m = c->lanes[lane].mapper;
  long long total = 0;
  int rc = export_sizes(c, m, ALOAM_EXPORT_MAP, &total); if (rc) return rc;
  if (total != n) return ALOAM_ERR_STATE;
  return n > 0 ? store_copy(c, c->d_export_layout, n, dst, device, false) : ALOAM_OK;
}

// Makes lane `lane`'s store (it exists) the one a validated snapshot table describes, with the snapshot's cube growth: *head
// (pinned host memory) goes to the device, k_store_import_tables rebuilds the tables and lays the store out, store_copy moves the
// head->n_points points of pts into the runs.  Synchronises.
int mapper_store_restore(aloam_ctx* c, int lane, const SnapStore* head, const char* pts, bool device, bool growth) {
  Mapper* m = c->lanes[lane].mapper;
  int ord[2];
  mapper_run_orders(c, growth, ord);
  if (!c->d_export_layout) CUDA_CHECK_RET(dalloc(c, &c->d_export_layout, 1));
  if (!c->d_snap_store) CUDA_CHECK_RET(dalloc(c, &c->d_snap_store, 1));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->d_snap_store, head, sizeof(SnapStore), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemsetAsync(m->frame.d_state, 0, sizeof(MapperState), c->stream));
  LAUNCH(c, KID_CUBES, k_store_import_tables, 1, 1024, 0, m->frame.d_state, c->d_snap_store, m->d_pts[0], m->d_pts[1], m->cap[0], m->cap[1], ord[0], ord[1],
         c->d_export_layout);
  if (head->n_points > 0) { const int rc = store_copy(c, c->d_export_layout, head->n_points, const_cast<char*>(pts), device, true); if (rc) return rc; }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

// The seeded records of a mapping frame (in[l].seed) on the current stream, two launches for all of them: k_store_seed_tables
// lays out record l's store as a copy of the prior map in c->d_seed_layout[l], k_store_seed_copy copies the map's points into it.
// Nothing is issued when no record seeds.
static int seed_stores(aloam_ctx* c, int nb, const MapperIn* in) {
  Batch<SeedLane> B = {};
  int n = 0;
  for (int l = 0; l < nb; ++l) {
    if (!in[l].seed) continue;
    const Lane& L = c->lanes[in[l].lane];
    const Mapper* m = L.mapper;
    B.a[n] = SeedLane{m->frame.d_state, {m->d_pts[0], m->d_pts[1]}, {m->cap[0], m->cap[1]}, c->d_seed_layout + n, {}};
    for (int k = 0; k < 7; ++k) B.a[n].init[k] = L.init[k];
    ++n;
  }
  if (n == 0) return ALOAM_OK;
  const PriorMap* P = c->prior;
  if (!P || !c->d_seed_layout) return ALOAM_ERR_STATE;   // an arming is dropped with the map it was checked against
  int ord[2];
  mapper_run_orders(c, c->cube_growth, ord);   // a seeded START is a mapped START: the context's cube growth
  LAUNCH(c, KID_CUBES, k_store_seed_tables, dim3(1, 1, n), 1024, 0, B, (const int*)P->d_cube_start, P->cen[0], P->cen[1], P->cen[2], ord[0], ord[1]);
  LAUNCH(c, KID_CUBES, k_store_seed_copy, dim3(std::min(kExportSegs, c->sms * 8), 1, n), 256, 0, (const ExportLayout*)P->d_layout, (const ExportLayout*)c->d_seed_layout);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

// One frame of alaserMapping's process() for nb trajectories ("lanes") on the current stream, entirely on the device: every launch
// covers all lanes, lane l in blockIdx.z, and each lane has its own cube store, stack filter buffers and registration set, so
// lane l computes exactly what a frame of lane l alone computes.  in[l]: the lane's less-sharp / less-flat clouds and their
// sizes, its odometry pose (7 doubles) and its output pose slot, all device pointers, the lane whose cube store record l
// runs on and whether that store starts a fresh trajectory; n_upper_* bound the cloud sizes of every lane.  Lane 0 registers
// with the context's set, shared with the host API.  A sharded job maps one lane.
int mapper_step_device(aloam_ctx* c, int nb, const MapperIn* in, int n_upper_c, int n_upper_s) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH || (nb > 1 && sharded_job(c))) return ALOAM_ERR_STATE;
  int rc = mapper_ensure(c, 0); if (rc) return rc;   // lane 0's store gives the sizes every lane shares
  for (int l = 0; l < nb; ++l) { rc = mapper_ensure(c, in[l].lane); if (rc) return rc; }
  rc = ensure_map_buffers(c); if (rc) return rc;     // lane 0's set
  const Mapper* m0 = c->lanes[0].mapper;
  Batch<MapperLane> B = {};
  MapLaneIO io[ALOAM_MAX_BATCH];
  SegFilter stack_f[ALOAM_MAX_BATCH], cube_f[ALOAM_MAX_BATCH];
  SegBuffers* bufs[ALOAM_MAX_BATCH];
  Batch<GridArgs> gs = {};
  unsigned fresh = 0;   // records whose store starts a new trajectory: reset by k_mapper_begin
  // index bits of a 50 m cube at the finer leaf: (50 / leaf + 3)^3 voxels at most (PCL itself gives up beyond 2^31)
  int cube_bits = 1;
  { const double side = std::floor(50.0 / std::min(c->cfg.line_res, c->cfg.plane_res)) + 3.0; const double cells = side * side * side;
    while (cube_bits < 31 && (double)(1ull << cube_bits) < cells) ++cube_bits; }
  for (int l = 0; l < nb; ++l) {   // record l runs on the store of lane in[l].lane
    Mapper* m = c->lanes[in[l].lane].mapper;
    MapperState* S = m->frame.d_state;
    const MapReg& reg = *m->frame.reg;
    MapperLane& a = B.a[l];
    a = frame_record(&m->frame, in[l], &stack_f[l], &bufs[l]);
    for (int t = 0; t < 2; ++t) { a.pts[t] = m->d_pts[t]; a.cap[t] = m->cap[t]; a.sub[t] = m->d_sub[t]; }
    a.world = m->d_world; a.cube = m->d_cube;
    if (in[l].fresh) fresh |= 1u << l;
    io[l] = MapLaneIO{reg, {m->d_sub[0], m->d_sub[1]}, S->stack_counts, S->x};
    gs.a[l] = GridArgs{reg.corner.grid, m->d_sub[0], &S->n_sub[0], reg.surf.grid, m->d_sub[1], &S->n_sub[1]};
    cube_f[l] = seg_filter(m->frame.buf, cube_bits, &S->err);
  }
  const int max_sub = m0->max_sub, cap1 = m0->cap[1];
  const int refilter_cap = (int)m0->frame.buf.cap;   // refilter_bound: the same for every lane
  int ord[2];                                  // the runs of the lanes that start a trajectory with this frame
  mapper_run_orders(c, c->cube_growth, ord);
  // ---- seeded STARTs: their stores become copies of the prior map, in order on this stream after the lanes' previous frames and
  //      before this frame's stack filters are forked, so nothing of the frame runs beside the seed
  rc = seed_stores(c, nb, in); if (rc) return rc;
  // ---- stack filters (:541-550), beside the gather + index build below, which read only the cube stores
  rc = stack_filters_fork(c, nb, B, stack_f, bufs, n_upper_c, n_upper_s); if (rc) return rc;
  launch_ex(c, KID_CUBES, k_mapper_begin, dim3(1, 1, nb), dim3(1024), 0, 1, true, B, max_sub, fresh, ord[0], ord[1]);
  launch_ex(c, KID_CUBES, k_mapper_gather, dim3(kMaxValid, 2, nb), dim3(256), 0, 1, true, B);
  if (c->shard_count > 1) {
    // A rank of a sharded job keeps the WHOLE cube store (the insertions below are replicated: the refined pose is bit-identical
    // on every rank) but indexes and searches only its x-slabs (+ halo) of the submap; the ranks meet in the all-reduce of the
    // normal equations inside the solve.  The too-thin test of k_mapper_prep is on the whole submap, the same on every rank.
    MapperState* S = m0->frame.d_state;
    rc = map_shard_index_device(c, m0->d_sub, S->n_sub, max_sub, &S->err); if (rc) return rc;
  } else {
    launch_ex(c, KID_MAP_GRID, k_grid_setup, dim3(1, 1, nb), dim3(32), 0, 1, true, gs);
    map_index_build(c, nb, io, max_sub);
  }
  c->have_map = true;
  CUDA_CHECK_RET(cudaStreamWaitEvent(c->stream, c->ev_stack_join, 0));   // join: the filtered stacks are ready
  launch_ex(c, KID_CUBES, k_mapper_prep, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  // ---- optimisation (:554-733)
  const int nq_upper = std::min(n_upper_c + n_upper_s, 2 * c->max_points);
  rc = map_register_device(c, nb, io, nq_upper, c->cfg.outer_iters); if (rc) return rc;
  launch_ex(c, KID_CUBES, k_mapper_update, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  // ---- insertion (:736-767)
  const int up = std::max(n_upper_c, n_upper_s);
  launch_ex(c, KID_CUBES, k_cube_ids, dim3(std::max(1, std::min((up + 255) / 256, std::max(1, c->sms * 2 / nb))), 2, nb), dim3(256), 0, 1, true, B, c->max_points);
  launch_ex(c, KID_CUBES, k_cube_insert, dim3(2, 1, nb), dim3(1024), (size_t)kInsertSmem, 1, true, B, c->max_points);
  // ---- per-cube re-filter of the valid cubes (:770-801): one segmented pass over <= 150 cubes of every lane, in place
  launch_ex(c, KID_CUBES, k_seg_cubes, dim3(1, 1, nb), dim3(256), 0, 1, true, B, c->cfg.line_res, c->cfg.plane_res, refilter_cap);
  vox_seg_filter(c, nb, cube_f, bufs, 2 * 75, refilter_cap, cap1);
  launch_ex(c, KID_CUBES, k_mapper_finish, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

// The high-frequency pose of nb skipped scans on the current stream, one launch: record l composes the T_wmap_wodom of lane
// in[l].lane's cube store (of its locator, when it localises) with in[l].odom7 into in[l].out7 (the clouds and `fresh` of in[l]
// are not read).  The lanes' stores or locators exist: a trajectory's first scan is always mapped.
int mapper_high_freq_device(aloam_ctx* c, int nb, const MapperIn* in) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH) return ALOAM_ERR_STATE;
  Batch<MapperLane> B = {};
  for (int l = 0; l < nb; ++l) {
    B.a[l].S = lane_frame(c, in[l].lane, in[l].localise)->d_state;
    B.a[l].odom7 = in[l].odom7;
    B.a[l].out7 = in[l].out7;
  }
  launch_ex(c, KID_CUBES, k_mapper_high_freq, dim3(1, 1, nb), dim3(32), 0, 1, false, B);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

// The registered full-resolution clouds of the nb lanes of the frame mapper_step_device has just issued, on the current stream
// (the mapper stream, before any later frame): record l moves the src[l] cloud of *n_full[l] points (device) by the refined pose of
// lane in[l].lane into dst[l].  n_upper bounds every cloud size.
int mapper_register_full_device(aloam_ctx* c, int nb, const MapperIn* in, const Pt4* const* src, const int* const* n_full, Pt4* const* dst, int n_upper) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH) return ALOAM_ERR_STATE;
  Batch<RegFullLane> B = {};
  for (int l = 0; l < nb; ++l) B.a[l] = RegFullLane{lane_frame(c, in[l].lane, in[l].localise)->d_state, src[l], n_full[l], dst[l]};
  const int blocks = std::max(1, std::min((n_upper + 255) / 256, std::max(1, c->sms * 2 / nb)));
  launch_ex(c, KID_CUBES, k_register_full, dim3(blocks, 1, nb), dim3(256), 0, 1, false, B);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

namespace {
// one record of k_map_rows: the frame state and the solve summaries of the frame a row's lane has just run, the row's slot, and
// the scoring points per type behind its score (0: the row is not scored)
struct MapRowLane {
  const MapperState* S;
  const LmSummary* summary;
  MapRowRec* row;
  int max_score;
};

// the rows of a frame's records, grid (1, 1, records) x 32 threads, after the frame's last kernel: thread t < outer copies the head
// of outer iteration t's summary, thread 0 the frame's flags, error word and sizes.  A scored row starts its count at 0 for the
// tracking score (k_inlier_score) and records the scoring points it covers.
__global__ void __launch_bounds__(32) k_map_rows(const __grid_constant__ Batch<MapRowLane> B, int outer) {
  const MapRowLane& a = B.a[blockIdx.z];
  const MapperState* S = a.S;
  MapRowRec* r = a.row;
  const int t = threadIdx.x;
  if (t < outer) {
    const LmSummary& s = a.summary[t];
    r->lm[t] = LmHead{s.termination, s.num_iterations, s.num_successful, s.num_jac_evals, s.n_edge, s.n_plane, s.initial_cost, s.final_cost};
  }
  if (t == 0) {
    r->flags = S->flags; r->err = S->frame_err; r->n_valid = S->n_valid;
    for (int k = 0; k < 2; ++k) { r->n_sub[k] = S->n_sub[k]; r->n_stack[k] = S->stack_counts[k]; }
    const int m = a.max_score > 0 ? scoring_points(S->stack_counts[0], S->stack_counts[1], a.max_score) : 0;
    r->score = a.max_score > 0 ? 0 : -1;
    r->n_score = m;
  }
}
}  // namespace

// k_map_rows over the nb records of the frame just issued on the current stream (the mapper stream, before the lanes' next
// frame): record l into rows[l]; its localising records are scored at max_score points per type (0: none is)
int map_rows_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, int max_score) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH) return ALOAM_ERR_STATE;
  Batch<MapRowLane> B = {};
  for (int l = 0; l < nb; ++l) {
    const LaneFrame* f = lane_frame(c, in[l].lane, in[l].localise);
    B.a[l] = MapRowLane{f->d_state, f->reg->summary, rows[l], in[l].localise ? max_score : 0};
  }
  LAUNCH(c, KID_MAP_ROWS, k_map_rows, dim3(1, 1, nb), 32, 0, B, std::min(c->cfg.outer_iters, 4));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

namespace {
// one record of k_recover_adopt: the localising lane's frame state, the row, the row's candidates and the best key k_reloc_topk
// left for them
struct RecoverAdopt {
  MapperState* S;
  MapRowRec* row;
  const double* cand;
  const unsigned long long* best;
};

// the last kernel of a recovery (recover.cu), one thread per record after k_reloc_topk: a triggered row records its best candidate
// (key = score << 32 | ~h) and adopts it when it beats the row's score and holds accept_frac of its scoring points -- transformUpdate
// at the candidate with the frame's odometry pose replaces the lane's T_wmap_wodom, which the lane's next frame hands off from.
// The row's map pose and frame state are left as the frame wrote them.
__global__ void __launch_bounds__(32) k_recover_adopt(const __grid_constant__ Batch<RecoverAdopt> B, int nb, float accept_frac) {
  const int l = threadIdx.x;
  if (l >= nb) return;
  const RecoverAdopt& a = B.a[l];
  MapRowRec* r = a.row;
  if (!r->rec_triggered) return;
  const unsigned long long key = a.best[0];
  const int h = (int)~(unsigned)(key & 0xffffffffull), s = (int)(key >> 32);
  const double* x = a.cand + (size_t)h * 7;
  const bool adopt = s > r->score && (float)s >= accept_frac * (float)r->n_score;
  r->rec_best = h;
  r->rec_best_score = s;
  r->rec_adopted = adopt;
  for (int k = 0; k < 7; ++k) r->rec_pose[k] = x[k];
  if (adopt) transform_update(a.S, x);
}
}  // namespace

// k_recover_adopt over the nb localising records of the frame just issued (recover.cu, after the candidates' scores and best keys):
// record l on its lane's locator, its row rows[l], candidates cand[l] and best key best[l]
int recover_adopt_device(aloam_ctx* c, int nb, const MapperIn* in, MapRowRec* const* rows, const double* const* cand,
                         const unsigned long long* const* best, float accept_frac) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH) return ALOAM_ERR_STATE;
  Batch<RecoverAdopt> B = {};
  for (int l = 0; l < nb; ++l) B.a[l] = RecoverAdopt{lane_frame(c, in[l].lane, in[l].localise)->d_state, rows[l], cand[l], best[l]};
  LAUNCH(c, KID_RECOVER_ADOPT, k_recover_adopt, 1, 32, 0, B, nb, accept_frac);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

int mapper_seed_ensure(aloam_ctx* c) {
  if (!c->d_seed_layout) CUDA_CHECK_RET(dalloc(c, &c->d_seed_layout, (size_t)c->n_lanes));
  return ALOAM_OK;
}

// Fills frame f of a new cube store or locator: its state and pinned mirror, a stack filter of filter_cap points and, unless it
// registers with `shared`, a registration set of `queries` points with grid tables of `slots` slots over submaps of `bound`
// points per type (map_reg_alloc; 0 slots: none).  f.mem takes the buffers only when every allocation succeeded; on a failure
// they are freed at once and f is to be discarded.
static int frame_alloc(aloam_ctx* c, LaneFrame& f, MapReg* shared, size_t queries, size_t bound, unsigned slots, size_t filter_cap) {
  BufGroup g;
  bool ok = stack_stream_ensure(c) == cudaSuccess && g.dev(&f.d_state, 1) && g.pinned(&f.h_state, 1);
  ok = ok && (shared || map_reg_alloc(g, &f.set, queries, bound, slots) == ALOAM_OK) && vox_seg_alloc(c, g, f.buf, filter_cap) == ALOAM_OK;
  if (!ok) { cudaGetLastError(); return ALOAM_ERR_CUDA; }
  f.mem = std::move(g);
  f.reg = shared ? shared : &f.set;
  return ALOAM_OK;
}

int mapper_ensure(aloam_ctx* c, int lane) {
  if (c->lanes[lane].mapper) return ALOAM_OK;
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  // lane 0 registers with the context's set, whose buffers ensure_map_buffers creates when they are first needed; another lane's
  // set is sized by the context's, which is created first
  if (lane > 0 && ensure_map_buffers(c) != ALOAM_OK) return ALOAM_ERR_CUDA;
  std::unique_ptr<Mapper> m(new (std::nothrow) Mapper());
  if (!m) return ALOAM_ERR_CUDA;
  mapper_slab_caps(c, m->cap);
  m->max_sub = c->cfg.max_map_points;
  const size_t mp = (size_t)c->max_points;
  BufGroup& g = m->mem;
  bool ok = true;
  for (int t = 0; t < 2 && ok; ++t) ok = g.dev(&m->d_pts[t], (size_t)kPool * m->cap[t]) && g.dev(&m->d_sub[t], (size_t)m->max_sub) && g.dev(&m->d_in[t], mp);
  ok = ok && g.dev(&m->d_world, 2 * mp) && g.dev(&m->d_cube, 2 * mp) && g.dev(&m->d_pose_io, 16);   // d_world: both stacks side by side
  ok = ok && cudaFuncSetAttribute(k_cube_insert, cudaFuncAttributeMaxDynamicSharedMemorySize, kInsertSmem) == cudaSuccess;
  if (!ok) { cudaGetLastError(); return ALOAM_ERR_CUDA; }
  int rc = frame_alloc(c, m->frame, lane == 0 ? &c->map : nullptr, 2 * mp, (size_t)c->max_map, (unsigned)c->map_slots, refilter_bound(m.get(), c));
  if (rc) return rc;
  rc = reset_lane(c, m.get());   // a lane is published with the state of a fresh trajectory, never uninitialised
  if (rc) return rc;
  Mapper* p = m.release();
  own(c, [p] { delete p; });
  c->lanes[lane].mapper = p;
  return ALOAM_OK;
}

// a new locator in *out, its state zeroed, published only when complete: a registration set without grid tables and a filter
// for the two scan stacks
int locator_create(aloam_ctx* c, LaneFrame** out) {
  std::unique_ptr<LaneFrame> f(new (std::nothrow) LaneFrame());
  if (!f) return ALOAM_ERR_CUDA;
  const size_t q = (size_t)2 * c->max_points;
  const int rc = frame_alloc(c, *f, nullptr, q, 0, 0, q); if (rc) return rc;
  if (cudaMemset(f->d_state, 0, sizeof(MapperState)) != cudaSuccess) { cudaGetLastError(); return ALOAM_ERR_CUDA; }
  LaneFrame* p = f.release();
  own(c, [p] { delete p; });
  *out = p;
  return ALOAM_OK;
}

// lane `lane`'s locator, created on first use
int locator_ensure(aloam_ctx* c, int lane) {
  return c->lanes[lane].locator ? ALOAM_OK : locator_create(c, &c->lanes[lane].locator);
}

LaneFrame* lane_frame(const aloam_ctx* c, int lane, bool localise) {
  const Lane& L = c->lanes[lane];
  return localise ? L.locator : L.mapper ? &L.mapper->frame : nullptr;
}

FrameView frame_view(const LaneFrame* f) {
  MapperState* S = f->d_state;
  return FrameView{{f->reg->stack[0], f->reg->stack[1]}, S->stack_counts, &S->flags, f->reg->summary, &S->err_acc};
}

PriorGrid prior_grid(const aloam_ctx* c) { return PriorGrid{c->prior->grid[0], c->prior->grid[1]}; }

int locator_stacks_device(aloam_ctx* c, LaneFrame* f, const MapperIn& in, int n_upper_c, int n_upper_s) {
  Batch<MapperLane> B = {};
  SegFilter sf;
  SegBuffers* bufs[1];
  B.a[0] = frame_record(f, in, &sf, &bufs[0]);
  const int rc = stack_filters_fork(c, 1, B, &sf, bufs, n_upper_c, n_upper_s); if (rc) return rc;
  CUDA_CHECK_RET(cudaStreamWaitEvent(c->stream, c->ev_stack_join, 0));
  return ALOAM_OK;
}

// One localising frame of nb records on the current stream: laserMapping.cpp:309-734 without the ring-buffer shift, against the
// context's prior map, which it only reads.  Record l as in mapper_step_device (in[l].lane is not read), run on the frame state
// and registration set of locator loc[l]; a record that starts a trajectory (in[l].fresh) begins from T_wmap_wodom init[l] (7
// doubles, host memory).  Every launch covers all records: the stack filters (forked, as the mapping frame's), k_locate_begin,
// the thin-map test, outer_iters x (k_map_knn5_prior, k_map_fit, LM), k_mapper_update, k_mapper_finish (the stack filter's error
// bit).
int locate_step_device(aloam_ctx* c, int nb, const MapperIn* in, LaneFrame* const* loc, const double* const* init, int n_upper_c, int n_upper_s) {
  const PriorMap* P = c->prior;
  if (nb < 1 || nb > ALOAM_MAX_BATCH || !P || sharded_job(c)) return ALOAM_ERR_STATE;
  Batch<MapperLane> B = {};
  Batch<LocateLane> L = {};
  MapLaneIO io[ALOAM_MAX_BATCH];
  SegFilter stack_f[ALOAM_MAX_BATCH];
  SegBuffers* bufs[ALOAM_MAX_BATCH];
  PriorSearch ps = {};
  ps.grid = PriorGrid{P->grid[0], P->grid[1]};
  for (int l = 0; l < nb; ++l) {
    MapperState* S = loc[l]->d_state;
    B.a[l] = frame_record(loc[l], in[l], &stack_f[l], &bufs[l]);
    L.a[l].S = S; L.a[l].odom7 = in[l].odom7; L.a[l].fresh = in[l].fresh;
    for (int k = 0; k < 7; ++k) L.a[l].init[k] = init[l][k];
    io[l] = MapLaneIO{*loc[l]->reg, {nullptr, nullptr}, S->stack_counts, S->x};
    ps.win[l][0] = S->sub_off[0]; ps.win[l][1] = S->sub_off[1]; ps.ctr[l] = S->ctr;
  }
  // the stack filters share s_stack with the mapping frame's: this fork is recorded after the whole mapping frame of the step
  int rc = stack_filters_fork(c, nb, B, stack_f, bufs, n_upper_c, n_upper_s); if (rc) return rc;
  launch_ex(c, KID_CUBES, k_locate_begin, dim3(1, 1, nb), dim3(256), 0, 1, true, L, (const int*)P->d_cube_start, P->cen[0], P->cen[1], P->cen[2]);
  CUDA_CHECK_RET(cudaStreamWaitEvent(c->stream, c->ev_stack_join, 0));   // join: the filtered stacks are ready
  launch_ex(c, KID_CUBES, k_mapper_prep, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  const int nq_upper = std::min(n_upper_c + n_upper_s, 2 * c->max_points);
  rc = map_register_device(c, nb, io, nq_upper, c->cfg.outer_iters, &ps); if (rc) return rc;
  launch_ex(c, KID_CUBES, k_mapper_update, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  launch_ex(c, KID_CUBES, k_mapper_finish, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

int locator_prior_search(aloam_ctx* c, int lane, PriorSearch* ps) {
  const PriorMap* P = c->prior;
  const Lane& L = c->lanes[lane];
  if (!P || !L.window) return ALOAM_ERR_STATE;
  MapperState* S = lane_frame(c, lane, true)->d_state;
  *ps = {};
  ps->grid = PriorGrid{P->grid[0], P->grid[1]};
  ps->win[0][0] = S->sub_off[0]; ps->win[0][1] = S->sub_off[1]; ps->ctr[0] = S->ctr;
  return ALOAM_OK;
}

// the digest of the context's prior map (it exists): on the first call one k_prior_digest launch over the whole map and one
// synchronisation, then the value kept with the map
static int prior_map_digest(aloam_ctx* c, unsigned long long* out) {
  PriorMap* P = c->prior;
  if (!P->have_digest) {
    if (!P->d_digest && !P->mem.dev(&P->d_digest, 1)) return ALOAM_ERR_CUDA;
    const long long n = (long long)P->n[0] + P->n[1];
    const int blocks = (int)std::max<long long>(1, std::min<long long>((n + kDigestThreads - 1) / kDigestThreads, (long long)c->sms * 8));
    CUDA_CHECK_RET(cudaMemsetAsync(P->d_digest, 0, sizeof(unsigned long long), c->stream));
    LAUNCH(c, KID_PRIOR_DIGEST, k_prior_digest, blocks, kDigestThreads, 0, P->cen[0], P->cen[1], P->cen[2], (const int*)P->d_cube_start,
           reinterpret_cast<const float4*>(P->pts[0]), P->n[0], reinterpret_cast<const float4*>(P->pts[1]), P->n[1], P->d_digest);
    unsigned long long d = 0;
    CUDA_CHECK_RET(cudaMemcpyAsync(&d, P->d_digest, sizeof(d), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
    CUDA_CHECK_RET(cudaGetLastError());
    prof_collect(c);
    P->digest = d;
    P->have_digest = true;
  }
  *out = P->digest;
  return ALOAM_OK;
}

int prior_map_identity(aloam_ctx* c, int cen[3], long long n[2], unsigned long long* digest) {
  const PriorMap* P = c->prior;
  if (!P) return ALOAM_ERR_STATE;
  for (int a = 0; a < 3; ++a) cen[a] = P->cen[a];
  for (int t = 0; t < 2; ++t) n[t] = P->n[t];
  return prior_map_digest(c, digest);
}

int locator_map_pose(aloam_ctx* c, int lane, double* dst) {
  const MapperState* S = lane_frame(c, lane, true)->d_state;
  CUDA_CHECK_RET(cudaMemcpyAsync(dst, S->q_wmap_wodom, 4 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(dst + 4, S->t_wmap_wodom, 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  return ALOAM_OK;
}

int locator_restore(aloam_ctx* c, int lane, const double T[7]) {
  const PriorMap* P = c->prior;
  MapperState* S = lane_frame(c, lane, true)->d_state;
  Pose7 p;
  for (int k = 0; k < 7; ++k) p.v[k] = T[k];
  CUDA_CHECK_RET(cudaMemsetAsync(S, 0, sizeof(MapperState), c->stream));
  LAUNCH(c, KID_CUBES, k_locate_restore, 1, 256, 0, S, p, P->cen[0], P->cen[1], P->cen[2]);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

extern "C" {

int aloam_prior_map_load(aloam_ctx* c, const void* blob, long long n_bytes) {
  if (!c || !blob || n_bytes < 0) return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c) || any_lane_localising(c)) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const int kind = snapshot_buffer_kind(c, blob);
  if (kind < 0) return ALOAM_ERR_INVALID_ARG;
  const char* b = static_cast<const char*>(blob);
  long long store = 0;
  int rc = snapshot_validate(c, b, n_bytes, kind, true, &store); if (rc) return rc;
  const SnapStore* H = c->h_snap_store;
  // ---- the new map is built beside the old one, which is replaced only when the new one is complete
  std::vector<int> cs((size_t)2 * (NCUBE + 1));
  for (int t = 0; t < 2; ++t) {
    long long run = 0;
    for (int i = 0; i < NCUBE; ++i) { cs[(size_t)t * (NCUBE + 1) + i] = (int)run; run += std::max(H->count[t][i], 0); }   // (<= 1024 slabs of <= 65536 points)
    cs[(size_t)t * (NCUBE + 1) + NCUBE] = (int)run;
  }
  return prior_install(c, H->cen, cs, [&](PriorMap* p) {
    return H->n_points > 0 ? store_copy(c, p->d_layout, H->n_points, const_cast<char*>(b) + store + sizeof(SnapStore), kind, true) : ALOAM_OK;
  });
}

int aloam_prior_map_build(aloam_ctx* c, aloam_cloud_view corner, aloam_cloud_view surf, const int centre[3], long long dropped[2]) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner); if (rc) return rc;
  rc = check_view(surf); if (rc) return rc;
  const int cen[3] = {centre ? centre[0] : 10, centre ? centre[1] : 10, centre ? centre[2] : 5};
  for (int a = 0; a < 3; ++a) if (cen[a] < -(1 << 20) || cen[a] > (1 << 20)) return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c) || any_lane_localising(c)) return ALOAM_ERR_STATE;
  // a cloud of more than 2^30 points, or two that together leave no room for a tile of the sort in int, cannot be indexed
  if (corner.n > (1 << 30) || surf.n > (1 << 30) || (long long)corner.n + surf.n > (long long)INT_MAX - 4096) return ALOAM_ERR_CAPACITY;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const int n = corner.n + surf.n, tiles = (n + kBuildTile - 1) / kBuildTile;
  const int blocks = std::max(1, std::min(tiles, c->sms * 8));
  std::vector<int> rank(kBuildSegs + 1, 0);
  int drop[2] = {0, 0};
  BuildScratch B(c->stream);
  if (!B.alloc((size_t)n, tiles)) return ALOAM_ERR_CUDA;
  if (n > 0) {
    rc = upload_cloud(c, corner, B.pts, n); if (rc) return rc;
    rc = upload_cloud(c, surf, B.pts + corner.n, surf.n); if (rc) return rc;
    CUDA_CHECK_RET(cudaMemcpyAsync(B.n_dev, &n, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, KID_PRIOR_BUILD, k_build_init, (kBuildSegs + 255) / 256, 256, 0, B.cnt, B.bbox, B.dropped);
    LAUNCH(c, KID_PRIOR_BUILD, k_build_classify, blocks, 256, 0, B.pts, corner.n, n, cen[0], cen[1], cen[2], B.seg, B.cnt, B.bbox, B.dropped);
    LAUNCH(c, KID_PRIOR_BUILD, k_build_params, 1, 1024, 0, B.cnt, B.bbox, c->cfg.line_res, c->cfg.plane_res, B.par, B.off);
    LAUNCH(c, KID_PRIOR_BUILD, k_build_keys, blocks, 256, 0, B.pts, n, B.seg, B.par, B.vox, B.keys[0], B.vals[0]);
    // stable: by voxel index (4 passes), then by segment (2 passes); both results end in buffer 0
    rc = vox_radix_sort(c, KID_PRIOR_BUILD, B.keys[0], B.vals[0], B.keys[1], B.vals[1], B.n_dev, n, 32, B.hist); if (rc) return rc;
    LAUNCH(c, KID_PRIOR_BUILD, k_build_gather, blocks, 256, 0, B.seg, n, B.keys[0], B.vals[0]);
    rc = vox_radix_sort(c, KID_PRIOR_BUILD, B.keys[0], B.vals[0], B.keys[1], B.vals[1], B.n_dev, n, 16, B.hist); if (rc) return rc;
    LAUNCH(c, KID_PRIOR_BUILD, k_build_heads, tiles, kBuildTile, 0, B.keys[0], B.vals[0], n, B.vox, B.par, B.head, B.tile_heads);
    LAUNCH(c, KID_PRIOR_BUILD, k_build_scan, 1, 1024, 0, B.tile_heads, tiles, B.total);
    LAUNCH(c, KID_PRIOR_BUILD, k_build_ranks, kBuildSegs + 1, 32, 0, B.off, B.head, B.tile_heads, B.total, n, B.rank);
    // the one synchronisation before the map exists: its sizes, every cube's, and the drops
    CUDA_CHECK_RET(cudaMemcpyAsync(rank.data(), B.rank, rank.size() * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(drop, B.dropped, sizeof(drop), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
    CUDA_CHECK_RET(cudaGetLastError());
  }
  const int n0 = rank[NCUBE];
  // a filtered cube: at most 65536 points while cube growth is off, ALOAM_MAX_CUBE_POINTS (the 18-bit rank of prior_tag) while on
  const int limit = c->cube_growth ? ALOAM_MAX_CUBE_POINTS : 65536;
  std::vector<int> cs((size_t)2 * (NCUBE + 1));
  for (int t = 0; t < 2; ++t)
    for (int i = 0; i <= NCUBE; ++i) {
      const int r = rank[(size_t)t * NCUBE + i] - (t ? n0 : 0);
      cs[(size_t)t * (NCUBE + 1) + i] = r;
      if (i > 0 && r - cs[(size_t)t * (NCUBE + 1) + i - 1] > limit) return ALOAM_ERR_CAPACITY;
    }
  rc = prior_install(c, cen, cs, [&](PriorMap* p) {
    if (n > 0) LAUNCH(c, KID_PRIOR_BUILD, k_build_emit, tiles, kBuildTile, 0, B.pts, B.keys[0], B.vals[0], n, B.par, B.head, B.tile_heads, n0, p->pts[0], p->pts[1]);
    return cudaGetLastError() == cudaSuccess ? ALOAM_OK : ALOAM_ERR_CUDA;
  });
  prof_collect(c);
  if (rc) return rc;
  if (dropped) { dropped[0] = drop[0]; dropped[1] = drop[1]; }
  return ALOAM_OK;
}

int aloam_prior_map_digest(aloam_ctx* c, unsigned long long* out) {
  if (!c || !out) return ALOAM_ERR_INVALID_ARG;
  if (!c->prior) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  return prior_map_digest(c, out);
}

int aloam_prior_map_clear(aloam_ctx* c) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  if (any_lane_localising(c)) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  prior_map_release(c);
  for (Lane& L : c->lanes) L.sched.arm = ARM_NONE;   // an arming needs a map
  return ALOAM_OK;
}

int aloam_lane_localise(aloam_ctx* c, int lane, const double q_init[4], const double t_init[3]) {
  if (!c || lane < 0 || lane >= c->n_lanes || !q_init || !t_init) return ALOAM_ERR_INVALID_ARG;
  double init[7];
  if (!map_pose_normalise(q_init, t_init, init)) return ALOAM_ERR_INVALID_ARG;
  if (!c->prior) return ALOAM_ERR_STATE;
  Lane& L = c->lanes[lane];
  for (int k = 0; k < 7; ++k) L.init[k] = init[k];
  L.sched.arm = ARM_LOCALISE;
  return ALOAM_OK;
}

int aloam_lane_map_on_prior(aloam_ctx* c, int lane, const double q_init[4], const double t_init[3]) {
  if (!c || lane < 0 || lane >= c->n_lanes || !q_init || !t_init) return ALOAM_ERR_INVALID_ARG;
  double init[7];
  if (!map_pose_normalise(q_init, t_init, init)) return ALOAM_ERR_INVALID_ARG;
  const PriorMap* P = c->prior;
  if (!P || sharded_job(c)) return ALOAM_ERR_STATE;
  // the START's map position is init's translation (identity odometry pose): its first frame's shift loop must end
  if (!map_position_fits(init + 4, P->cen)) return ALOAM_ERR_INVALID_ARG;
  // every cube within its ceiling and every run in the pool, under the context's cube growth now: one slab per cube while it is
  // off, the runs store_import_body packs while it is on
  int cap[2], ord[2];
  mapper_slab_caps(c, cap);
  mapper_run_orders(c, c->cube_growth, ord);
  for (int t = 0; t < 2; ++t)
    if (P->max_cube[t] > (cap[t] << ord[t]) || (c->cube_growth ? P->run_slabs[t] : P->n_cubes[t]) > kPool) return ALOAM_ERR_CAPACITY;
  Lane& L = c->lanes[lane];
  for (int k = 0; k < 7; ++k) L.init[k] = init[k];
  L.sched.arm = ARM_MAP_ON_PRIOR;
  return ALOAM_OK;
}

int aloam_set_cube_growth(aloam_ctx* c, int on) {
  if (!c || (on != 0 && on != 1)) return ALOAM_ERR_INVALID_ARG;
  c->cube_growth = on != 0;
  for (Lane& L : c->lanes) if (L.sched.arm == ARM_MAP_ON_PRIOR) L.sched.arm = ARM_NONE;   // its fit was checked under the old setting
  return ALOAM_OK;
}

}  // extern "C"

extern "C" {

int aloam_mapper_reset(aloam_ctx* c) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const bool fresh = !c->lanes[0].mapper;
  int rc = mapper_ensure(c, 0); if (rc) return rc;   // a new lane 0 is reset already
  for (size_t l = fresh ? 1 : 0; l < c->lanes.size(); ++l)   // every lane that exists
    if (c->lanes[l].mapper) { rc = reset_lane(c, c->lanes[l].mapper); if (rc) return rc; }
  return ALOAM_OK;
}

int aloam_mapper_step(aloam_ctx* c, aloam_cloud_view corner_last, aloam_cloud_view surf_last, const double q_wodom_curr[4],
                      const double t_wodom_curr[3], double q_w_curr[4], double t_w_curr[3], aloam_stats* stats) {
  if (!c || !q_wodom_curr || !t_wodom_curr || !q_w_curr || !t_w_curr) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_last); if (rc) return rc;
  rc = check_view(surf_last); if (rc) return rc;
  if (corner_last.n > c->max_points || surf_last.n > c->max_points) return ALOAM_ERR_CAPACITY;   // before any state is touched
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  rc = mapper_ensure(c, 0); if (rc) return rc;
  Mapper* m = c->lanes[0].mapper;
  CUDA_CHECK_RET(cudaEventRecord(c->ev0, c->stream));
  // the inputs are uploaded to mapper-owned device buffers first: the views may alias any ctx-owned pinned buffer
  rc = upload_cloud(c, corner_last, m->d_in[0], c->max_points); if (rc) return rc;
  rc = upload_cloud(c, surf_last, m->d_in[1], c->max_points); if (rc) return rc;
  c->pin->mapper_counts[0] = corner_last.n; c->pin->mapper_counts[1] = surf_last.n;
  CUDA_CHECK_RET(cudaMemcpyAsync(m->frame.d_state->in_counts, c->pin->mapper_counts, 8, cudaMemcpyHostToDevice, c->stream));
  for (int k = 0; k < 4; ++k) c->pin->mapper_pose_in[k] = q_wodom_curr[k];
  for (int k = 0; k < 3; ++k) c->pin->mapper_pose_in[4 + k] = t_wodom_curr[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(m->d_pose_io, c->pin->mapper_pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  const MapperIn one{m->d_in[0], &m->frame.d_state->in_counts[0], m->d_in[1], &m->frame.d_state->in_counts[1], m->d_pose_io, m->d_pose_io + 7, 0, 0};
  rc = peer_err_reset(c); if (rc) return rc;
  rc = mapper_step_device(c, 1, &one, corner_last.n, surf_last.n);
  if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->mapper_pose_out, m->d_pose_io + 7, 56, cudaMemcpyDeviceToHost, c->stream));
  rc = peer_err_fetch(c, &c->pin->peer_err); if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, m->frame.reg->summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(&m->frame.h_state->flags, &m->frame.d_state->flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaEventRecord(c->ev1, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  for (int k = 0; k < 4; ++k) q_w_curr[k] = c->pin->mapper_pose_out[k];
  for (int k = 0; k < 3; ++k) t_w_curr[k] = c->pin->mapper_pose_out[4 + k];
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  frame_stats_from(c->h_summary, stats, c->cfg.outer_iters, m->frame.h_state->flags, ms);
  if (m->frame.h_state->frame_err & 1) return ALOAM_ERR_CAPACITY;   // a voxel index range beyond the key width: results would be wrong
  if (c->pin->peer_err) return ALOAM_ERR_COMM;                // a peer did not answer: the pose rests on a partial sum
  return ALOAM_OK;
}

int aloam_mapper_debug_state_lane(aloam_ctx* c, int lane, int centre[3], int* n_valid, int valid[125], double q_wmap_wodom[4],
                                  double t_wmap_wodom[3], long long totals[2]) {
  if (!c) return ALOAM_ERR_STATE;
  if (lane < 0 || lane >= ALOAM_MAX_BATCH) return ALOAM_ERR_INVALID_ARG;
  if (lane >= c->n_lanes) return ALOAM_ERR_STATE;   // no such lane, so no store
  // a lane whose trajectory localises answers from its locator, with the totals of the prior map it reads
  const Lane& L = c->lanes[lane];
  const bool loc = L.sched.localising && L.locator && c->prior;
  const LaneFrame* f = lane_frame(c, lane, loc);
  if (!f) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaMemcpy(f->h_state, f->d_state, sizeof(MapperState), cudaMemcpyDeviceToHost));
  const MapperState* h = f->h_state;
  if (centre) for (int a = 0; a < 3; ++a) centre[a] = h->cen[a];
  if (n_valid) *n_valid = h->n_valid;
  if (valid) for (int i = 0; i < h->n_valid && i < 125; ++i) valid[i] = h->valid[i];
  if (q_wmap_wodom) for (int k = 0; k < 4; ++k) q_wmap_wodom[k] = h->q_wmap_wodom[k];
  if (t_wmap_wodom) for (int k = 0; k < 3; ++k) t_wmap_wodom[k] = h->t_wmap_wodom[k];
  if (totals && loc) { for (int t = 0; t < 2; ++t) totals[t] = c->prior->n[t]; }
  else if (totals)
    for (int t = 0; t < 2; ++t) {
      totals[t] = 0;
      for (int i = 0; i < NCUBE; ++i) { const int s = h->slab_of[t][i]; if (s >= 0) totals[t] += h->cnt[t][s]; }
    }
  return ALOAM_OK;
}

int aloam_mapper_debug_state(aloam_ctx* c, int centre[3], int* n_valid, int valid[125], double q_wmap_wodom[4], double t_wmap_wodom[3],
                             long long totals[2]) {
  return aloam_mapper_debug_state_lane(c, 0, centre, n_valid, valid, q_wmap_wodom, t_wmap_wodom, totals);
}

int aloam_mapper_debug_cube_lane(aloam_ctx* c, int lane, int which, int cube, aloam_cloud_view* out) {
  if (!c || !out || which < 0 || which > 1 || cube < 0 || cube >= NCUBE || lane < 0 || lane >= ALOAM_MAX_BATCH) return ALOAM_ERR_INVALID_ARG;
  if (lane >= c->n_lanes || !c->lanes[lane].mapper) return ALOAM_ERR_STATE;
  Mapper* m = c->lanes[lane].mapper;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaMemcpy(m->frame.h_state, m->frame.d_state, sizeof(MapperState), cudaMemcpyDeviceToHost));
  const int s = m->frame.h_state->slab_of[which][cube];
  const int n = s < 0 ? 0 : m->frame.h_state->cnt[which][s];
  // a cube beyond max_points (cube growth) is read into a pinned buffer of ALOAM_MAX_CUBE_POINTS points, created on first use
  if (n > c->max_points && !c->h_cube) CUDA_CHECK_RET(halloc(c, &c->h_cube, (size_t)ALOAM_MAX_CUBE_POINTS));
  Pt4* h = n > c->max_points ? c->h_cube : c->h_out[4];
  out->data = reinterpret_cast<const float*>(h); out->n = n; out->stride_floats = 4;
  if (n > 0) CUDA_CHECK_RET(cudaMemcpy(h, m->d_pts[which] + (size_t)s * m->cap[which], (size_t)n * sizeof(Pt4), cudaMemcpyDeviceToHost));
  return ALOAM_OK;
}

int aloam_mapper_export(aloam_ctx* c, int lane, int what, float* out, long long capacity, long long* n_out) {
  if (!c || !n_out || capacity < 0 || lane < ALOAM_PRIOR_MAP || lane >= ALOAM_MAX_BATCH) return ALOAM_ERR_INVALID_ARG;
  if (what != ALOAM_EXPORT_SURROUND && what != ALOAM_EXPORT_MAP) return ALOAM_ERR_INVALID_ARG;
  const bool prior = lane == ALOAM_PRIOR_MAP;
  if (prior && what != ALOAM_EXPORT_MAP) return ALOAM_ERR_INVALID_ARG;   // the prior map has no frame, so no surround
  const Mapper* m = prior || lane >= c->n_lanes ? nullptr : c->lanes[lane].mapper;
  const PriorMap* pm = c->prior;
  if (prior ? !pm : !m) return ALOAM_ERR_STATE;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  long long n = 0;
  int rc = ALOAM_OK;
  if (prior) n = (long long)pm->n[0] + pm->n[1];
  else { rc = export_sizes(c, m, what, &n); if (rc) return rc; }
  *n_out = n;
  if (!out && capacity == 0) return ALOAM_OK;   // the size only
  if (!out) return ALOAM_ERR_INVALID_ARG;
  if (capacity < n) return ALOAM_ERR_CAPACITY;
  if (n == 0) return ALOAM_OK;
  cudaPointerAttributes at = {};
  CUDA_CHECK_RET(cudaPointerGetAttributes(&at, out));
  const bool device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
  rc = store_copy(c, prior ? pm->d_layout : c->d_export_layout, n, reinterpret_cast<char*>(out), device, false); if (rc) return rc;
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

int aloam_mapper_debug_cube(aloam_ctx* c, int which, int cube, aloam_cloud_view* out) {
  if (!c || !c->lanes[0].mapper) return ALOAM_ERR_INVALID_ARG;
  return aloam_mapper_debug_cube_lane(c, 0, which, cube, out);
}

int aloam_debug_seg_voxel_filter(aloam_ctx* c, const aloam_cloud_view* segs, const float* leaves, int n_segs, int idx_bits, float* out,
                                 int* out_counts, int* err) {
  if (!c || n_segs < 0 || (n_segs > 0 && (!segs || !leaves || !out_counts)) || !err || idx_bits < 1 || idx_bits > 31) return ALOAM_ERR_INVALID_ARG;
  if (n_segs > ALOAM_MAX_SEGS) return ALOAM_ERR_CAPACITY;
  size_t total = 0;
  int per_seg = 0;
  for (int s = 0; s < n_segs; ++s) {
    int rc = check_view(segs[s]); if (rc) return rc;
    if (!(leaves[s] > 0.f)) return ALOAM_ERR_INVALID_ARG;
    total += (size_t)segs[s].n;
    per_seg = std::max(per_seg, segs[s].n);
  }
  if (total > 0 && !out) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  int rc = mapper_ensure(c, 0); if (rc) return rc;
  Mapper* m = c->lanes[0].mapper;
  if (total > m->frame.buf.cap) return ALOAM_ERR_CAPACITY;
  if (!m->d_dbg_err) {   // first use: the group is published complete
    BufGroup g;
    Pt4* pts;
    int *counts, *e;
    if (!g.dev(&pts, m->frame.buf.cap) || !g.dev(&counts, ALOAM_MAX_SEGS) || !g.dev(&e, 1)) return ALOAM_ERR_CUDA;
    m->dbg = std::move(g);
    m->d_dbg_pts = pts; m->d_dbg_counts = counts; m->d_dbg_err = e;
  }
  // the segments back to back, filtered in place like the cubes of the re-filter; the mapper state is not touched (the
  // descriptors, offsets and sort buffers are scratch that every frame rewrites before use)
  SegDesc desc[ALOAM_MAX_SEGS];
  int counts[ALOAM_MAX_SEGS];
  size_t off = 0;
  for (int s = 0; s < n_segs; ++s) {
    rc = upload_cloud(c, segs[s], m->d_dbg_pts + off, (int)(m->frame.buf.cap - off)); if (rc) return rc;
    desc[s] = SegDesc{m->d_dbg_pts + off, m->d_dbg_counts + s, leaves[s], m->d_dbg_pts + off, m->d_dbg_counts + s};
    counts[s] = segs[s].n;
    off += (size_t)segs[s].n;
  }
  if (n_segs > 0) {
    CUDA_CHECK_RET(cudaMemcpyAsync(m->frame.buf.segs, desc, sizeof(SegDesc) * n_segs, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(m->d_dbg_counts, counts, sizeof(int) * n_segs, cudaMemcpyHostToDevice, c->stream));
  }
  CUDA_CHECK_RET(cudaMemcpyAsync(m->frame.buf.n_seg, &n_segs, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemsetAsync(m->d_dbg_err, 0, sizeof(int), c->stream));
  if (n_segs > 0) {
    const SegFilter f = seg_filter(m->frame.buf, idx_bits, m->d_dbg_err);
    SegBuffers* bp = &m->frame.buf;
    vox_seg_filter(c, 1, &f, &bp, n_segs, (int)std::max<size_t>(total, 1), std::max(per_seg, 1));
  }
  CUDA_CHECK_RET(cudaGetLastError());
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  if (n_segs > 0) CUDA_CHECK_RET(cudaMemcpy(out_counts, m->d_dbg_counts, sizeof(int) * n_segs, cudaMemcpyDeviceToHost));
  CUDA_CHECK_RET(cudaMemcpy(err, m->d_dbg_err, sizeof(int), cudaMemcpyDeviceToHost));
  off = 0;
  for (int s = 0; s < n_segs; ++s) {
    if (out_counts[s] > 0)
      CUDA_CHECK_RET(cudaMemcpy(out + 4 * off, m->d_dbg_pts + off, (size_t)out_counts[s] * sizeof(Pt4), cudaMemcpyDeviceToHost));
    off += (size_t)segs[s].n;
  }
  return ALOAM_OK;
}

}  // extern "C"
