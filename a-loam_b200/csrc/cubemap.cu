// Map cube store of alaserMapping and the per-frame loop around it -- replaces laserMapping.cpp:74-108 (state),
// :142-163 (pose hand-off, pointAssociateToMap), :309-550 (centre cube, ring-buffer shift, 75-cube gather, stack
// filters) and :736-801 (insertion, per-cube VoxelGrid).  SURVEY.md section 8 f-1 / f-2.
//
// Second version: the WHOLE frame runs on the device without a host synchronisation, so it can sit at the end of the scan
// stream (aloam_scan_stream_mapped) or behind the host API (aloam_mapper_step, one sync at the end to return the pose):
//   * state (T_wmap_wodom, centre offsets, cube -> slab table, per-slab counts, slab free list) lives in device memory;
//   * k_mapper_begin : transformAssociateToMap, centre cube, ring-buffer shift (the reference rotates 4851 smart pointers;
//                      here one CTA permutes the cube -> slab table, one thread per line of cubes, and returns the slabs
//                      of the cubes that scroll out to the free list), valid-cube list in the reference's i, j, k order;
//   * k_mapper_gather: the <= 75 valid cubes device-to-device into the submap, then the hash-grid build of mapping.cu;
//   * the two scan-stack filters as ONE segmented VoxelGrid (voxel.cu), the registration of mapping.cu on device views;
//   * k_mapper_update: transformUpdate, refined pose out;
//   * k_cube_ids / k_cube_insert: pointAssociateToMap + cube of the stored point, then a STABLE append (push_back order =
//                      stack order): one CTA walks the stack in chunks, warps take turns, __match_any groups the lanes of a
//                      cube and the group leader advances the cube's running end (allocating a slab from the free list
//                      for a cube that was empty) -- O(n) instead of the O(n^2 / 256) rank search of the first version;
//   * the per-cube re-filter of the valid cubes as ONE segmented VoxelGrid over up to 150 segments, in place.
// Slabs are a POOL (1024 per cloud type, 16 k corner / 64 k surf points each: 1.3 GB) handed out on the device on first
// insertion, not 4851 x 2 slabs (6.4 GB) up front.  A full slab or an exhausted pool drops the overflow and raises
// ALOAM_FLAG_CUBE_OVERFLOW instead of failing the frame (the reference grows its cubes without bound between re-filters).
#include <climits>
#include "common.cuh"
#include "ctx.h"

namespace {

constexpr int CW = 21, CH = 21, CD = 11, NCUBE = CW * CH * CD;   // laserCloudWidth / Height / Depth (:77-82)
constexpr int kMaxValid = 128;
constexpr int kPool = 1024;                                      // physical slabs per cloud type

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
  int err;                                   // of the running frame -- bit 0: voxel index range, bit 1: slab overflow, bit 2: pool
                                             // exhausted, bit 3: submap capacity; cleared when the frame ends
  int err_acc;                               // OR of the frames' words over one aloam_scan_stream_mapped call
  int frames;
  int zero, sink;                            // always 0 (count of a cube without a slab) ; write-only dummy
  int free_top;                              // slabs [free_top, kPool) of free_list are free ... per type
  int free_top2;
  int slab_of[2][NCUBE];                     // cube -> slab of that type, -1 = none
  int cnt[2][kPool];                         // points per slab
  int free_list[2][kPool];
};

struct Mapper {
  int cap[2] = {0, 0};
  Pt4* d_pts[2] = {nullptr, nullptr};       // [kPool * cap] slabs
  Pt4* d_sub[2] = {nullptr, nullptr};       // gathered submap
  Pt4* d_in[2] = {nullptr, nullptr};        // host API: uploaded less-sharp / less-flat clouds
  Pt4* d_world = nullptr;                   // insertion scratch: transformed stack points
  int* d_cube = nullptr;                    //                    their cube index (-1 = outside the ring buffer)
  MapperState* d_state = nullptr;
  MapperState* h_state = nullptr;           // pinned mirror (debug / host API read-back)
  SegBuffers buf;                           // the segmented filter of the stack filters and the per-cube re-filter
  double* d_pose_io = nullptr;              // [14] host API: odometry pose in, refined pose out
  Pt4* d_dbg_pts = nullptr;                 // aloam_debug_seg_voxel_filter: segments back to back [buf.cap] ...
  int* d_dbg_counts = nullptr;              //                                their sizes [ALOAM_MAX_SEGS]
  int* d_dbg_err = nullptr;                 //                                private error word
  int max_sub = 0;
  MapReg* reg = nullptr;                    // registration set: lane 0 shares the context's with the host API, the others own one
  cudaStream_t s_aux = nullptr;             // the stack filters run here, beside the submap gather + index build
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
};

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

// ---- Eigen-order quaternion helpers (operation order of Eigen::Quaternion: the pose hand-off is compared bit for bit)
struct Qd { double x, y, z, w; };
__host__ __device__ inline Qd qmul(const Qd& a, const Qd& b) {
  Qd r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
__host__ __device__ inline Qd qinv(const Qd& a) {
  const double n2 = a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
  return Qd{-a.x / n2, -a.y / n2, -a.z / n2, a.w / n2};
}
__host__ __device__ inline void qrot(const Qd& q, const double v[3], double o[3]) {
  double uv[3] = {q.y * v[2] - q.z * v[1], q.z * v[0] - q.x * v[2], q.x * v[1] - q.y * v[0]};
  uv[0] = uv[0] + uv[0]; uv[1] = uv[1] + uv[1]; uv[2] = uv[2] + uv[2];
  const double c2[3] = {q.y * uv[2] - q.z * uv[1], q.z * uv[0] - q.x * uv[2], q.x * uv[1] - q.y * uv[0]};
  o[0] = v[0] + q.w * uv[0] + c2[0]; o[1] = v[1] + q.w * uv[1] + c2[1]; o[2] = v[2] + q.w * uv[2] + c2[2];
}

// int((v + 25.0) / 50.0) + centre, minus one when v + 25.0 < 0   (:314-325, :741-750)
__host__ __device__ inline int cube_coord(double v, int centre) {
  int c = int((v + 25.0) / 50.0) + centre;
  if (v + 25.0 < 0) c--;
  return c;
}
__host__ __device__ inline int cube_index(int i, int j, int k) { return i + CW * j + CW * CH * k; }

// :327-509 -- one step of the ring buffer along `axis` for the line (u, v) of this thread; towards_high: every cube moves one
// index up, the top cube wraps to index 0 and is emptied (its slabs go back to the free lists)
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
      const int slot = atomicSub(ty == 0 ? &S->free_top : &S->free_top2, 1) - 1;   // push
      S->free_list[ty][slot] = wrapped;
    }
  }
}

// the state of a fresh trajectory (laserMapping.cpp:74-117): identity T_wmap_wodom, centre cube (10, 10, 5), every slab free
// and no cube holding one.  Run by all threads of one CTA.  It leaves alone the word of the call (err_acc) and every field the
// stack filter writes while k_mapper_begin runs beside it (stack_counts, err, in_counts): between frames `err` is 0 already
// (k_mapper_finish), and reset_lane zeroes the whole state before it runs this.
__device__ void mapper_fresh_state(MapperState* S) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = tid; i < NCUBE; i += nt) { S->slab_of[0][i] = -1; S->slab_of[1][i] = -1; }
  for (int i = tid; i < kPool; i += nt) { S->cnt[0][i] = 0; S->cnt[1][i] = 0; S->free_list[0][i] = i; S->free_list[1][i] = i; }
  for (int i = tid; i < kMaxValid; i += nt) S->valid[i] = 0;
  for (int i = tid; i < 2 * (kMaxValid + 1); i += nt) S->sub_off[i / (kMaxValid + 1)][i % (kMaxValid + 1)] = 0;
  if (tid == 0) {
    for (int k = 0; k < 4; ++k) { S->q_wmap_wodom[k] = k == 3 ? 1.0 : 0.0; S->q_wodom[k] = 0.0; }
    for (int k = 0; k < 3; ++k) { S->t_wmap_wodom[k] = 0.0; S->t_wodom[k] = 0.0; S->ctr[k] = 0; }
    for (int k = 0; k < 7; ++k) S->x[k] = 0.0;
    S->cen[0] = 10; S->cen[1] = 10; S->cen[2] = 5;
    S->n_valid = 0; S->n_sub[0] = 0; S->n_sub[1] = 0;
    S->flags = 0; S->frame_err = 0; S->frames = 0; S->zero = 0; S->sink = 0;
    S->free_top = 0; S->free_top2 = 0;
  }
}
// grid (1): the host-side reset of one lane (reset_lane)
__global__ void __launch_bounds__(1024) k_mapper_reset(MapperState* S) { mapper_fresh_state(S); }

// transformAssociateToMap (:142-146), centre cube + shift (:314-509), valid cubes (:511-529), gather offsets
__device__ __forceinline__ void mapper_begin_body(MapperState* S, const double* __restrict__ odom7, int max_sub, bool fresh) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (fresh) {   // the lane starts a new trajectory with this frame: no extra launch, in order on the mapper stream
    mapper_fresh_state(S);
    __syncthreads();
  }
  __shared__ int s_ctr[3], s_cen[3];
  const int tid = threadIdx.x;
  if (tid == 0) {
    const Qd qm{S->q_wmap_wodom[0], S->q_wmap_wodom[1], S->q_wmap_wodom[2], S->q_wmap_wodom[3]};
    const Qd qo{odom7[0], odom7[1], odom7[2], odom7[3]};
    const double to[3] = {odom7[4], odom7[5], odom7[6]};
    const Qd q0 = qmul(qm, qo);
    double r[3]; qrot(qm, to, r);
    S->x[0] = q0.x; S->x[1] = q0.y; S->x[2] = q0.z; S->x[3] = q0.w;
    S->x[4] = r[0] + S->t_wmap_wodom[0]; S->x[5] = r[1] + S->t_wmap_wodom[1]; S->x[6] = r[2] + S->t_wmap_wodom[2];
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
// grid (1, 1, lanes); bit l of `fresh`: record l starts a new trajectory with this frame, its state is reset first
__global__ void __launch_bounds__(1024) k_mapper_begin(const __grid_constant__ Batch<MapperLane> B, int max_sub, unsigned fresh) {
  const MapperLane& a = B.a[blockIdx.z];
  mapper_begin_body(a.S, a.odom7, max_sub, (fresh >> blockIdx.z) & 1u);
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


// transformUpdate (:148-152) ; refined pose out
__device__ __forceinline__ void mapper_update_body(MapperState* S, double* __restrict__ out7) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x || blockIdx.x) return;
  const Qd qw{S->x[0], S->x[1], S->x[2], S->x[3]};
  const Qd qo{S->q_wodom[0], S->q_wodom[1], S->q_wodom[2], S->q_wodom[3]};
  const Qd qn = qmul(qw, qinv(qo));
  double r[3]; qrot(qn, S->t_wodom, r);
  S->q_wmap_wodom[0] = qn.x; S->q_wmap_wodom[1] = qn.y; S->q_wmap_wodom[2] = qn.z; S->q_wmap_wodom[3] = qn.w;
  S->t_wmap_wodom[0] = S->x[4] - r[0]; S->t_wmap_wodom[1] = S->x[5] - r[1]; S->t_wmap_wodom[2] = S->x[6] - r[2];
  if (out7) for (int k = 0; k < 7; ++k) out7[k] = S->x[k];
  S->frames++;
}
__global__ void k_mapper_update(const __grid_constant__ Batch<MapperLane> B) {   // grid (1, 1, lanes)
  const MapperLane& a = B.a[blockIdx.z];
  mapper_update_body(a.S, a.out7);
}


// end of the frame, after insertion and re-filter have set their error bits: slab overflow, pool exhaustion and submap
// truncation become this frame's ALOAM_FLAG_CUBE_OVERFLOW, the frame's word joins the per-call accumulation, and `err` starts
// the next frame clear (everything of the next frame -- the stack filter forked onto the auxiliary stream included -- is
// ordered after this kernel)
__device__ __forceinline__ void mapper_finish_body(MapperState* S) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  if (threadIdx.x || blockIdx.x) return;
  const int e = S->err;
  if (e & 14) S->flags |= ALOAM_FLAG_CUBE_OVERFLOW;
  S->frame_err = e;
  S->err_acc |= e;
  S->err = 0;
}
__global__ void k_mapper_finish(const __grid_constant__ Batch<MapperLane> B) { mapper_finish_body(B.a[blockIdx.z].S); }   // grid (1, 1, lanes)


// pointAssociateToMap (:154-163) in double, stored as float, then the cube of the stored point (:741-758)
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
    const Pt4 p = stack[i];
    const double vx = (double)p.x, vy = (double)p.y, vz = (double)p.z;
    double uvx = uy * vz - uz * vy, uvy = uz * vx - ux * vz, uvz = ux * vy - uy * vx;
    uvx = uvx + uvx; uvy = uvy + uvy; uvz = uvz + uvz;
    const double cx = uy * uvz - uz * uvy, cy = uz * uvx - ux * uvz, cz = ux * uvy - uy * uvx;
    Pt4 s;
    s.x = (float)(((vx + w * uvx) + cx) + tx);
    s.y = (float)(((vy + w * uvy) + cy) + ty);
    s.z = (float)(((vz + w * uvz) + cz) + tz);
    s.i = p.i;
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


// stable append of the stack points to their cubes (push_back order = stack order, :759-767).  ONE CTA per cloud (blockIdx.x: the
// corner and the surf store are independent, the two appends run side by side): the stack is walked in
// chunks of 1024; inside a chunk the warps take turns, the lanes of one cube form a group (__match_any) whose leader
// advances the cube's running end in shared memory -- and takes a slab from the free list when the cube had none.
__device__ __forceinline__ void cube_insert_body(const Pt4* __restrict__ world, const int* __restrict__ cube, int scratch_stride, MapperState* S,
                                                      Pt4* __restrict__ pts0, int cap0, Pt4* __restrict__ pts1, int cap1) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int ty = blockIdx.x;
  world += (size_t)ty * scratch_stride; cube += (size_t)ty * scratch_stride;
  Pt4* __restrict__ pts = ty ? pts1 : pts0;
  const int cap = ty ? cap1 : cap0;
  __shared__ int s_end[NCUBE];    // running end of every cube
  __shared__ int s_slab[NCUBE];   // cube -> slab (the warps' turns must not wait on global memory)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = S->stack_counts[ty];
  int* slab_of = S->slab_of[ty];
  int* cnt = S->cnt[ty];
  for (int c = tid; c < NCUBE; c += blockDim.x) { const int s = slab_of[c]; s_slab[c] = s; s_end[c] = s < 0 ? 0 : cnt[s]; }
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + tid;
    const int mine = i < n ? cube[i] : -1;
    const Pt4 p = i < n ? world[i] : Pt4{0.f, 0.f, 0.f, 0.f};
    const int warps = min(32, (n - base + 31) / 32);
    for (int w = 0; w < warps; ++w) {
      if (warp == w) {
        const unsigned grp = __match_any_sync(0xffffffffu, mine);
        const int leader = __ffs(grp) - 1;
        int start = 0, slab = -1;
        if (mine >= 0 && lane == leader) {
          slab = s_slab[mine];
          if (slab < 0) {   // first point of an empty cube: take a slab from the pool (several group leaders of one warp may do so at once)
            int* top = ty == 0 ? &S->free_top : &S->free_top2;
            const int idx = atomicAdd(top, 1);
            if (idx < kPool) { slab = S->free_list[ty][idx]; s_slab[mine] = slab; }
            else { atomicSub(top, 1); atomicOr(&S->err, 4); }
          }
          start = s_end[mine];
          s_end[mine] = start + __popc(grp);
        }
        start = __shfl_sync(0xffffffffu, start, leader);
        slab = __shfl_sync(0xffffffffu, slab, leader);
        if (mine >= 0 && slab >= 0) {
          const int pos = start + __popc(grp & ((1u << lane) - 1u));
          if (pos < cap) pts[(size_t)slab * cap + pos] = p;
          else atomicOr(&S->err, 2);   // slab full: the overflow is dropped (flagged), the frame goes on
        }
      }
      __syncthreads();
    }
  }
  for (int c = tid; c < NCUBE; c += blockDim.x) { const int s = s_slab[c]; if (s >= 0) { slab_of[c] = s; cnt[s] = min(s_end[c], cap); } }
}
// grid (2 clouds, 1, lanes): every CTA has its own shared cube tables and takes slabs from its lane's free list
__global__ void __launch_bounds__(1024) k_cube_insert(const __grid_constant__ Batch<MapperLane> B, int scratch_stride) {
  const MapperLane& a = B.a[blockIdx.z];
  cube_insert_body(a.world, a.cube, scratch_stride, a.S, a.pts[0], a.cap[0], a.pts[1], a.cap[1]);
}


// segment descriptors of the per-cube re-filter (:770-801): every valid cube that has a slab, corner cubes then surf cubes, in place
__device__ __forceinline__ void seg_cubes_body(MapperState* S, SegDesc* segs, int* n_seg, Pt4* p0, Pt4* p1, int cap0, int cap1, float leaf0, float leaf1) {
  pdl_launch_dependents();
  pdl_wait();   // may have been launched with a programmatic dependency on the previous kernel of the stream
  const int t = threadIdx.x, nv = S->n_valid;
  if (t < 2 * nv) {
    const int ty = t >= nv, v = ty ? t - nv : t;
    const int s = S->slab_of[ty][S->valid[v]];
    Pt4* base = s < 0 ? (ty ? p1 : p0) : (ty ? p1 : p0) + (size_t)s * (ty ? cap1 : cap0);
    int* np = s < 0 ? &S->zero : &S->cnt[ty][s];
    segs[t] = SegDesc{base, np, ty ? leaf1 : leaf0, base, s < 0 ? &S->sink : np};
  }
  if (t == 0) { *n_seg = 2 * nv; S->zero = 0; }
}
// grid (1, 1, lanes)
__global__ void __launch_bounds__(256) k_seg_cubes(const __grid_constant__ Batch<MapperLane> B, float leaf0, float leaf1) {
  const MapperLane& a = B.a[blockIdx.z];
  seg_cubes_body(a.S, a.segs, a.n_seg, a.pts[0], a.pts[1], a.cap[0], a.cap[1], leaf0, leaf1);
}


// points one segmented filter can sort: the re-filter takes every point of the <= 75 valid cubes of each type, full slabs
// included (the submap gather truncates only its own copy at max_map_points), the stack filter two scan clouds
size_t refilter_bound(const Mapper* m, const aloam_ctx* c) {
  return std::max((size_t)75 * (m->cap[0] + m->cap[1]), (size_t)2 * c->max_points);
}

// the state of a fresh trajectory (mapper_fresh_state, the routine k_mapper_begin runs for a lane that starts one), with the
// fields that routine leaves alone zeroed first
int reset_lane(aloam_ctx* c, Mapper* m) {
  CUDA_CHECK_RET(cudaMemsetAsync(m->d_state, 0, sizeof(MapperState), c->stream));
  LAUNCH(c, KID_CUBES, k_mapper_reset, 1, 1024, 0, m->d_state);
  CUDA_CHECK_RET(cudaGetLastError());
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  return ALOAM_OK;
}

int ensure_mapper(aloam_ctx* c, int lane) {
  if (c->mapper[lane]) return ALOAM_OK;
  if (c->cfg.max_map_points <= 0) return ALOAM_ERR_CAPACITY;
  Mapper* m = new (std::nothrow) Mapper();
  if (!m) return ALOAM_ERR_CUDA;
  own(c, [m] { delete m; });
  m->cap[0] = std::min(16384, c->max_points);
  m->cap[1] = std::min(65536, c->max_points);
  m->max_sub = c->cfg.max_map_points;
  bool ok = true;
  for (int t = 0; t < 2 && ok; ++t) {
    ok = ok && dalloc(c, &m->d_pts[t], (size_t)kPool * m->cap[t]) == cudaSuccess;
    ok = ok && dalloc(c, &m->d_sub[t], (size_t)m->max_sub) == cudaSuccess;
    ok = ok && dalloc(c, &m->d_in[t], (size_t)c->max_points) == cudaSuccess;
  }
  ok = ok && dalloc(c, &m->d_world, (size_t)2 * c->max_points) == cudaSuccess;   // both stacks side by side
  ok = ok && dalloc(c, &m->d_cube, (size_t)2 * c->max_points) == cudaSuccess;
  ok = ok && dalloc(c, &m->d_state, 1) == cudaSuccess;
  ok = ok && halloc(c, &m->h_state, 1) == cudaSuccess;
  ok = ok && dalloc(c, &m->d_pose_io, 16) == cudaSuccess;
  ok = ok && screate(c, &m->s_aux) == cudaSuccess;
  ok = ok && ecreate(c, &m->ev_fork, cudaEventDisableTiming) == cudaSuccess && ecreate(c, &m->ev_join, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && vox_seg_alloc(c, m->buf, refilter_bound(m, c)) == ALOAM_OK;
  // lane 0's set is the context's, whose buffers ensure_map_buffers creates when they are first needed; another lane's set is
  // created here, after the context's (which fixes the table size)
  m->reg = lane == 0 ? &c->map : new (std::nothrow) MapReg();
  if (lane > 0 && m->reg) own(c, [r = m->reg] { delete r; });
  ok = ok && m->reg && (lane == 0 || (ensure_map_buffers(c) == ALOAM_OK && map_reg_alloc(c, m->reg) == ALOAM_OK));
  if (!ok) {   // publish nothing half-built: what was acquired belongs to the context until aloam_destroy
    cudaGetLastError();
    return ALOAM_ERR_CUDA;
  }
  const int rc = reset_lane(c, m);   // a lane is published with the state of a fresh trajectory, never uninitialised
  if (rc) return rc;
  c->mapper[lane] = m;
  return ALOAM_OK;
}

}  // namespace

// One frame of alaserMapping's process() for nb trajectories ("lanes") on the current stream, entirely on the device: every launch
// covers all lanes, lane l in blockIdx.z, and each lane has its own cube store, stack filter buffers and registration set, so
// lane l computes exactly what a frame of lane l alone computes.  in[l]: the lane's less-sharp / less-flat clouds and their
// sizes, its odometry pose (7 doubles) and its output pose slot, all device pointers, the lane whose cube store record l
// runs on and whether that store starts a fresh trajectory; n_upper_* bound the cloud sizes of every lane.  Lane 0 registers
// with the context's set, shared with the host API.  A sharded job maps one lane.
int mapper_step_device(aloam_ctx* c, int nb, const MapperIn* in, int n_upper_c, int n_upper_s) {
  if (nb < 1 || nb > ALOAM_MAX_BATCH || (nb > 1 && sharded_job(c))) return ALOAM_ERR_STATE;
  int rc = ensure_mapper(c, 0); if (rc) return rc;   // lane 0's auxiliary stream carries the stack filters of every lane
  for (int l = 0; l < nb; ++l) { rc = ensure_mapper(c, in[l].lane); if (rc) return rc; }
  rc = ensure_map_buffers(c); if (rc) return rc;     // lane 0's set
  Mapper* m0 = static_cast<Mapper*>(c->mapper[0]);
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
    const int lane = in[l].lane;
    Mapper* m = static_cast<Mapper*>(c->mapper[lane]);
    MapperState* S = m->d_state;
    const MapReg& reg = *m->reg;
    B.a[l] = MapperLane{S, in[l].odom7, in[l].out7, {m->d_pts[0], m->d_pts[1]}, {m->cap[0], m->cap[1]}, {m->d_sub[0], m->d_sub[1]}, {in[l].corner, in[l].surf},
                        {in[l].nc, in[l].ns}, {reg.stack[0], reg.stack[1]}, m->d_world, m->d_cube, m->buf.segs, m->buf.n_seg};
    if (in[l].fresh) fresh |= 1u << l;
    io[l] = MapLaneIO{reg, {m->d_sub[0], m->d_sub[1]}, S->stack_counts, S->x};
    gs.a[l] = GridArgs{reg.corner.grid, m->d_sub[0], &S->n_sub[0], reg.surf.grid, m->d_sub[1], &S->n_sub[1]};
    stack_f[l] = seg_filter(m->buf, 31, &S->err);
    cube_f[l] = seg_filter(m->buf, cube_bits, &S->err);
    bufs[l] = &m->buf;
  }
  const int max_sub = m0->max_sub, cap1 = m0->cap[1];
  const int refilter_cap = (int)m0->buf.cap;   // refilter_bound: the same for every lane
  // ---- stack filters (:541-550): one segmented pass for both clouds of every lane.  They read only the scans' clouds, the
  // gather + index build below only the cube stores: two independent chains, the filters forked onto an auxiliary stream and
  // joined before the registration.
  {
    cudaStream_t main_stream = c->stream;
    CUDA_CHECK_RET(cudaEventRecord(m0->ev_fork, main_stream));
    CUDA_CHECK_RET(cudaStreamWaitEvent(m0->s_aux, m0->ev_fork, 0));
    c->stream = m0->s_aux;
    launch_ex(c, KID_VOXEL, k_seg_two, dim3(1, 1, nb), dim3(32), 0, 1, false, B, c->cfg.line_res, c->cfg.plane_res);
    vox_seg_filter(c, nb, stack_f, bufs, 2, n_upper_c + n_upper_s, std::max(n_upper_c, n_upper_s));
    const cudaError_t e = cudaEventRecord(m0->ev_join, m0->s_aux);
    c->stream = main_stream;
    CUDA_CHECK_RET(e);
  }
  launch_ex(c, KID_CUBES, k_mapper_begin, dim3(1, 1, nb), dim3(1024), 0, 1, true, B, max_sub, fresh);
  launch_ex(c, KID_CUBES, k_mapper_gather, dim3(kMaxValid, 2, nb), dim3(256), 0, 1, true, B);
  if (c->shard_count > 1) {
    // A rank of a sharded job keeps the WHOLE cube store (the insertions below are replicated: the refined pose is bit-identical
    // on every rank) but indexes and searches only its x-slabs (+ halo) of the submap; the ranks meet in the all-reduce of the
    // normal equations inside the solve.  The too-thin test of k_mapper_prep is on the whole submap, the same on every rank.
    MapperState* S = m0->d_state;
    rc = map_shard_index_device(c, m0->d_sub, S->n_sub, max_sub, &S->err); if (rc) return rc;
  } else {
    launch_ex(c, KID_MAP_GRID, k_grid_setup, dim3(1, 1, nb), dim3(32), 0, 1, true, gs);
    map_index_build(c, nb, io, max_sub);
  }
  c->have_map = true;
  CUDA_CHECK_RET(cudaStreamWaitEvent(c->stream, m0->ev_join, 0));   // join: the filtered stacks are ready
  launch_ex(c, KID_CUBES, k_mapper_prep, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  // ---- optimisation (:554-733)
  const int nq_upper = std::min(n_upper_c + n_upper_s, 2 * c->max_points);
  rc = map_register_device(c, nb, io, nq_upper); if (rc) return rc;
  launch_ex(c, KID_CUBES, k_mapper_update, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  // ---- insertion (:736-767)
  const int up = std::max(n_upper_c, n_upper_s);
  launch_ex(c, KID_CUBES, k_cube_ids, dim3(std::max(1, std::min((up + 255) / 256, std::max(1, c->sms * 2 / nb))), 2, nb), dim3(256), 0, 1, true, B, c->max_points);
  launch_ex(c, KID_CUBES, k_cube_insert, dim3(2, 1, nb), dim3(1024), 0, 1, true, B, c->max_points);
  // ---- per-cube re-filter of the valid cubes (:770-801): one segmented pass over <= 150 cubes of every lane, in place
  launch_ex(c, KID_CUBES, k_seg_cubes, dim3(1, 1, nb), dim3(256), 0, 1, true, B, c->cfg.line_res, c->cfg.plane_res);
  vox_seg_filter(c, nb, cube_f, bufs, 2 * 75, refilter_cap, cap1);
  launch_ex(c, KID_CUBES, k_mapper_finish, dim3(1, 1, nb), dim3(32), 0, 1, true, B);
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

// the per-call error accumulation of a mapped stream call (device word; the lane's mapper must exist)
int* mapper_err_acc(aloam_ctx* c, int lane) { return &static_cast<Mapper*>(c->mapper[lane])->d_state->err_acc; }

// the cube stores of lanes 0 .. nb-1, each created on first use with the state of a fresh trajectory.  A failure leaves the
// lanes that existed untouched.
int mapper_ensure_lanes(aloam_ctx* c, int nb) {
  for (int l = 0; l < nb; ++l) { int rc = ensure_mapper(c, l); if (rc) return rc; }
  return ALOAM_OK;
}

extern "C" {

int aloam_mapper_reset(aloam_ctx* c) {
  if (!c) return ALOAM_ERR_INVALID_ARG;
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const bool fresh = c->mapper[0] == nullptr;
  int rc = ensure_mapper(c, 0); if (rc) return rc;   // a new lane 0 is reset already
  for (int l = fresh ? 1 : 0; l < ALOAM_MAX_BATCH; ++l)   // every lane that exists
    if (c->mapper[l]) { rc = reset_lane(c, static_cast<Mapper*>(c->mapper[l])); if (rc) return rc; }
  return ALOAM_OK;
}

int aloam_mapper_step(aloam_ctx* c, aloam_cloud_view corner_last, aloam_cloud_view surf_last, const double q_wodom_curr[4],
                      const double t_wodom_curr[3], double q_w_curr[4], double t_w_curr[3], aloam_stats* stats) {
  if (!c || !q_wodom_curr || !t_wodom_curr || !q_w_curr || !t_w_curr) return ALOAM_ERR_INVALID_ARG;
  int rc = check_view(corner_last); if (rc) return rc;
  rc = check_view(surf_last); if (rc) return rc;
  if (corner_last.n > c->max_points || surf_last.n > c->max_points) return ALOAM_ERR_CAPACITY;   // before any state is touched
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  rc = mapper_ensure_lanes(c, 1); if (rc) return rc;
  Mapper* m = static_cast<Mapper*>(c->mapper[0]);
  CUDA_CHECK_RET(cudaEventRecord(c->ev0, c->stream));
  // the inputs are uploaded to mapper-owned device buffers first: the views may alias any ctx-owned pinned buffer
  rc = upload_cloud(c, corner_last, m->d_in[0], c->max_points); if (rc) return rc;
  rc = upload_cloud(c, surf_last, m->d_in[1], c->max_points); if (rc) return rc;
  c->pin->mapper_counts[0] = corner_last.n; c->pin->mapper_counts[1] = surf_last.n;
  CUDA_CHECK_RET(cudaMemcpyAsync(m->d_state->in_counts, c->pin->mapper_counts, 8, cudaMemcpyHostToDevice, c->stream));
  for (int k = 0; k < 4; ++k) c->pin->mapper_pose_in[k] = q_wodom_curr[k];
  for (int k = 0; k < 3; ++k) c->pin->mapper_pose_in[4 + k] = t_wodom_curr[k];
  CUDA_CHECK_RET(cudaMemcpyAsync(m->d_pose_io, c->pin->mapper_pose_in, 56, cudaMemcpyHostToDevice, c->stream));
  const MapperIn one{m->d_in[0], &m->d_state->in_counts[0], m->d_in[1], &m->d_state->in_counts[1], m->d_pose_io, m->d_pose_io + 7, 0, 0};
  rc = peer_err_reset(c); if (rc) return rc;
  rc = mapper_step_device(c, 1, &one, corner_last.n, surf_last.n);
  if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->mapper_pose_out, m->d_pose_io + 7, 56, cudaMemcpyDeviceToHost, c->stream));
  rc = peer_err_fetch(c, &c->pin->peer_err); if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(c->h_summary, m->reg->summary, sizeof(LmSummary) * 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(&m->h_state->flags, &m->d_state->flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaEventRecord(c->ev1, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  prof_collect(c);
  for (int k = 0; k < 4; ++k) q_w_curr[k] = c->pin->mapper_pose_out[k];
  for (int k = 0; k < 3; ++k) t_w_curr[k] = c->pin->mapper_pose_out[4 + k];
  float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
  if (m->h_state->flags & ALOAM_FLAG_MAP_TOO_THIN) { if (stats) { std::memset(stats, 0, sizeof(*stats)); stats->flags = m->h_state->flags; stats->ms_total = ms; } }
  else fill_stats(c, stats, c->cfg.outer_iters, m->h_state->flags, ms);
  if (m->h_state->frame_err & 1) return ALOAM_ERR_CAPACITY;   // a voxel index range beyond the key width: results would be wrong
  if (c->pin->peer_err) return ALOAM_ERR_COMM;                // a peer did not answer: the pose rests on a partial sum
  return ALOAM_OK;
}

int aloam_mapper_debug_state_lane(aloam_ctx* c, int lane, int centre[3], int* n_valid, int valid[125], double q_wmap_wodom[4],
                                  double t_wmap_wodom[3], long long totals[2]) {
  if (!c) return ALOAM_ERR_STATE;
  if (lane < 0 || lane >= ALOAM_MAX_BATCH) return ALOAM_ERR_INVALID_ARG;
  if (!c->mapper[lane]) return ALOAM_ERR_STATE;
  Mapper* m = static_cast<Mapper*>(c->mapper[lane]);
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaMemcpy(m->h_state, m->d_state, sizeof(MapperState), cudaMemcpyDeviceToHost));
  const MapperState* h = m->h_state;
  if (centre) for (int a = 0; a < 3; ++a) centre[a] = h->cen[a];
  if (n_valid) *n_valid = h->n_valid;
  if (valid) for (int i = 0; i < h->n_valid && i < 125; ++i) valid[i] = h->valid[i];
  if (q_wmap_wodom) for (int k = 0; k < 4; ++k) q_wmap_wodom[k] = h->q_wmap_wodom[k];
  if (t_wmap_wodom) for (int k = 0; k < 3; ++k) t_wmap_wodom[k] = h->t_wmap_wodom[k];
  if (totals)
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
  if (!c->mapper[lane]) return ALOAM_ERR_STATE;
  Mapper* m = static_cast<Mapper*>(c->mapper[lane]);
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  CUDA_CHECK_RET(cudaMemcpy(m->h_state, m->d_state, sizeof(MapperState), cudaMemcpyDeviceToHost));
  const int s = m->h_state->slab_of[which][cube];
  const int n = s < 0 ? 0 : m->h_state->cnt[which][s];
  out->data = reinterpret_cast<const float*>(c->h_out[4]); out->n = n; out->stride_floats = 4;
  if (n > 0) CUDA_CHECK_RET(cudaMemcpy(c->h_out[4], m->d_pts[which] + (size_t)s * m->cap[which], (size_t)n * sizeof(Pt4), cudaMemcpyDeviceToHost));
  return ALOAM_OK;
}

int aloam_mapper_debug_cube(aloam_ctx* c, int which, int cube, aloam_cloud_view* out) {
  if (!c || !c->mapper[0]) return ALOAM_ERR_INVALID_ARG;
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
  int rc = mapper_ensure_lanes(c, 1); if (rc) return rc;
  Mapper* m = static_cast<Mapper*>(c->mapper[0]);
  if (total > m->buf.cap) return ALOAM_ERR_CAPACITY;
  if (!m->d_dbg_err) {   // first use; the pointer that marks the group as ready is allocated last
    CUDA_CHECK_RET(dalloc(c, &m->d_dbg_pts, m->buf.cap));
    CUDA_CHECK_RET(dalloc(c, &m->d_dbg_counts, ALOAM_MAX_SEGS));
    CUDA_CHECK_RET(dalloc(c, &m->d_dbg_err, 1));
  }
  // the segments back to back, filtered in place like the cubes of the re-filter; the mapper state is not touched (the
  // descriptors, offsets and sort buffers are scratch that every frame rewrites before use)
  SegDesc desc[ALOAM_MAX_SEGS];
  int counts[ALOAM_MAX_SEGS];
  size_t off = 0;
  for (int s = 0; s < n_segs; ++s) {
    rc = upload_cloud(c, segs[s], m->d_dbg_pts + off, (int)(m->buf.cap - off)); if (rc) return rc;
    desc[s] = SegDesc{m->d_dbg_pts + off, m->d_dbg_counts + s, leaves[s], m->d_dbg_pts + off, m->d_dbg_counts + s};
    counts[s] = segs[s].n;
    off += (size_t)segs[s].n;
  }
  if (n_segs > 0) {
    CUDA_CHECK_RET(cudaMemcpyAsync(m->buf.segs, desc, sizeof(SegDesc) * n_segs, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(cudaMemcpyAsync(m->d_dbg_counts, counts, sizeof(int) * n_segs, cudaMemcpyHostToDevice, c->stream));
  }
  CUDA_CHECK_RET(cudaMemcpyAsync(m->buf.n_seg, &n_segs, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemsetAsync(m->d_dbg_err, 0, sizeof(int), c->stream));
  if (n_segs > 0) {
    const SegFilter f = seg_filter(m->buf, idx_bits, m->d_dbg_err);
    SegBuffers* bp = &m->buf;
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
