// Lane snapshots (include/aloam_b200.h: aloam_lane_save, aloam_lane_save_localising, aloam_lane_restore, aloam_snapshot_check):
// everything later scans of a lane of aloam_scan_stream_lanes depend on, written out and read back exactly, so a trajectory can be
// suspended and resumed in any lane of any context with the same result-affecting configuration.  A lane's state between two
// stream calls:
//   - its warm start and world pose (Lane::d_pose, d_world);
//   - its "last" less-sharp / less-flat clouds, in feature slot (frame - 1) mod kFeatSlots -- the slot the next step reads as
//     "last" -- whose search index is rebuilt from the clouds on restore;
//   - the index of its next scan and its mode (LaneSched::scan, mapped, localising);
//   - mapped (format 1): its cube store, in the slab-free form of SnapStore (cubemap.cu saves and restores it);
//   - localising (format 2): its locator's T_wmap_wodom -- the one field of the frame state a later frame, skipped row, row record
//     or recovery reads before writing it -- and the name of the prior map it localises against (centre, sizes, digest), which a
//     restore checks against the context's own map.
// Formats: snapshot.h.
#include <climits>
#include <cmath>
#include <cstring>
#include "common.cuh"
#include "ctx.h"
#include "quat.cuh"

namespace {

constexpr char kMagic[8] = {'A', 'L', 'O', 'A', 'M', 'L', 'S', '1'};
constexpr int kMaxCentre = 1 << 20;    // |cen[a]|: the range aloam_prior_map_build accepts
constexpr int kCubeSlack = 16;         // cubes the map position may lie outside the buffer on an axis (the shift loop's steps)

bool all_finite(const double* v, int n) {
  for (int k = 0; k < n; ++k) if (!std::isfinite(v[k])) return false;
  return true;
}

// the cube coordinate of map coordinate v under centre offset `centre` (laserMapping.cpp:314-325), with the range check of
// build_cube_coord (cubemap.cu): false when (v + 25) / 50 is not finite or lies beyond int
bool centre_cube(double v, int centre, long long* out) {
  const double s = v + 25.0;
  const double q = s / 50.0;
  if (!(q > -2147483649.0 && q < 2147483648.0)) return false;
  *out = (long long)(int)q + centre - (s < 0 ? 1 : 0);
  return true;
}

// byte offset of the store section (the end of the unmapped snapshot; the locator section of a format-2 one)
long long store_offset(const SnapHeader& h) { return (long long)sizeof(SnapHeader) + 16ll * ((long long)h.n_less_sharp + h.n_less_flat); }

bool localising(const SnapHeader& h) { return h.version == kSnapVersionLocalise; }

// the header on its own: magic, version, sizes of the sections before the store table.  n_bytes must be what the header says
// the snapshot holds; a mapped snapshot must hold its store table at least, a format-2 one exactly its locator section.
int check_header(const SnapHeader& h, long long n_bytes) {
  if (std::memcmp(h.magic, kMagic, 8) != 0 || (h.version != kSnapVersion && h.version != kSnapVersionLocalise)) return ALOAM_ERR_SNAPSHOT;
  if ((h.mapped != 0 && h.mapped != 1) || h.scan_index < 1 || h.n_less_sharp < 0 || h.n_less_flat < 0) return ALOAM_ERR_SNAPSHOT;
  if (h.ring_source != ALOAM_RING_ELEVATION && h.ring_source != ALOAM_RING_FIELD) return ALOAM_ERR_SNAPSHOT;
  if (h.cube_growth != 0 && h.cube_growth != 1) return ALOAM_ERR_SNAPSHOT;
  if (h.total_bytes != n_bytes) return ALOAM_ERR_SNAPSHOT;
  if (!all_finite(h.warm, 7) || !all_finite(h.world, 7)) return ALOAM_ERR_SNAPSHOT;
  if (localising(h))   // a localising lane has no cube store of its own
    return !h.mapped && !h.cube_growth && n_bytes == store_offset(h) + (long long)sizeof(SnapLocalise) ? ALOAM_OK : ALOAM_ERR_SNAPSHOT;
  if (!h.mapped) return n_bytes == store_offset(h) ? ALOAM_OK : ALOAM_ERR_SNAPSHOT;
  if (h.slab_cap[0] < 1 || h.slab_cap[1] < 1 || h.max_map_points < 1) return ALOAM_ERR_SNAPSHOT;
  return n_bytes >= store_offset(h) + (long long)sizeof(SnapStore) ? ALOAM_OK : ALOAM_ERR_SNAPSHOT;
}

// the store table of a mapped snapshot whose header passed check_header: centre offsets within +-2^20, a finite T_wmap_wodom, a
// map position T_wmap_wodom * world whose centre cube lies at most kCubeSlack cubes outside the buffer on every axis (the next
// frame's shift loop runs one pass per cube beyond the edge: an unbounded position would never end it), the valid list, every
// count within its ceiling under the snapshot's cube growth (the slab capacity while off, the largest run's while on), the runs
// the counts need (store_import_body: one slab up to the slab capacity, else the next power of two of ceil(n / cap)) at most
// kSnapPool slabs per type -- with every run one slab: at most kSnapPool cubes of a type hold a slab --, and a payload of exactly
// the counted points that ends the snapshot
int check_store(const SnapHeader& h, const SnapStore& s) {
  for (int a = 0; a < 3; ++a) if (s.cen[a] < -kMaxCentre || s.cen[a] > kMaxCentre) return ALOAM_ERR_SNAPSHOT;
  if (!all_finite(s.q_wmap_wodom, 4) || !all_finite(s.t_wmap_wodom, 3)) return ALOAM_ERR_SNAPSHOT;
  {
    const Qd qm{s.q_wmap_wodom[0], s.q_wmap_wodom[1], s.q_wmap_wodom[2], s.q_wmap_wodom[3]};
    double p[3];
    qrot(qm, h.world + 4, p);
    for (int a = 0; a < 3; ++a) p[a] += s.t_wmap_wodom[a];
    if (!map_position_fits(p, s.cen)) return ALOAM_ERR_SNAPSHOT;
  }
  if (s.n_valid < 0 || s.n_valid > 125) return ALOAM_ERR_SNAPSHOT;
  for (int v = 0; v < s.n_valid; ++v)
    if (s.valid[v] < 0 || s.valid[v] >= kSnapCubes) return ALOAM_ERR_SNAPSHOT;
  long long points = 0;
  for (int ty = 0; ty < 2; ++ty) {
    const long long cap = h.slab_cap[ty];
    long long top = cap;   // the largest run's capacity: the largest power of two r <= kSnapPool with r cap <= ALOAM_MAX_CUBE_POINTS
    for (int r = 2; h.cube_growth && r <= kSnapPool && r * cap <= ALOAM_MAX_CUBE_POINTS; r *= 2) top = r * cap;
    long long slabs = 0;
    for (int i = 0; i < kSnapCubes; ++i) {
      const int n = s.count[ty][i];
      if (n < -1 || n > top) return ALOAM_ERR_SNAPSHOT;
      if (n < 0) continue;
      long long run = 1;
      while (run * cap < n) run *= 2;
      slabs += run; points += n;
    }
    if (slabs > kSnapPool) return ALOAM_ERR_SNAPSHOT;
  }
  if (s.n_points != points) return ALOAM_ERR_SNAPSHOT;
  return h.total_bytes == store_offset(h) + (long long)sizeof(SnapStore) + 16 * points ? ALOAM_OK : ALOAM_ERR_SNAPSHOT;
}

// the locator section of a format-2 snapshot whose header passed check_header: a finite T_wmap_wodom with a quaternion that is not
// zero, centre offsets within +-2^20, point counts >= 0, and a map position T_wmap_wodom * world (translation) whose
// (x + 25) / 50 is finite and within int, with its centre cube within int too (k_locate_begin's cube_coord is defined there; a
// position off the map only thins the window)
int check_localise(const SnapHeader& h, const SnapLocalise& s) {
  if (!all_finite(s.q_wmap_wodom, 4) || !all_finite(s.t_wmap_wodom, 3)) return ALOAM_ERR_SNAPSHOT;
  double n2 = 0;
  for (int k = 0; k < 4; ++k) n2 += s.q_wmap_wodom[k] * s.q_wmap_wodom[k];
  if (!(n2 > 0)) return ALOAM_ERR_SNAPSHOT;
  for (int a = 0; a < 3; ++a) if (s.centre[a] < -kMaxCentre || s.centre[a] > kMaxCentre) return ALOAM_ERR_SNAPSHOT;
  if (s.map_points[0] < 0 || s.map_points[1] < 0) return ALOAM_ERR_SNAPSHOT;
  const Qd qm{s.q_wmap_wodom[0], s.q_wmap_wodom[1], s.q_wmap_wodom[2], s.q_wmap_wodom[3]};
  double p[3];
  qrot(qm, h.world + 4, p);
  for (int a = 0; a < 3; ++a) {
    long long c = 0;
    if (!centre_cube(p[a] + s.t_wmap_wodom[a], s.centre[a], &c) || c < INT_MIN || c > INT_MAX) return ALOAM_ERR_SNAPSHOT;
  }
  return ALOAM_OK;
}

// the configuration fields of the header that can change a result
void fingerprint(const aloam_ctx* c, SnapHeader* h) {
  const aloam_config& g = c->cfg;
  h->n_scans = g.n_scans; h->ring_source = g.ring_source; h->distortion = g.distortion; h->mapping_skip_frame = g.mapping_skip_frame;
  h->outer_iters = g.outer_iters; h->inner_iters = g.inner_iters;
  h->minimum_range = g.minimum_range; h->line_res = g.line_res; h->plane_res = g.plane_res;
  mapper_slab_caps(c, h->slab_cap);
  h->max_map_points = g.max_map_points;
  h->huber = g.huber; h->dist_sq_thresh = g.dist_sq_thresh; h->nearby_scan = g.nearby_scan;
}

// the snapshot's configuration against the context's, bit patterns for the floating-point fields.  The scan-to-map fields count
// only for a mapped snapshot: an odometry-only trajectory moves between contexts that map differently (or not at all).  A
// localising one needs the fields a localising frame reads (the stack filters' leaves and which scans register); it has no
// store, so the slab capacities and max_map_points do not count.
bool same_config(const SnapHeader& s, const SnapHeader& c) {
  auto same = [](const void* a, const void* b, size_t n) { return std::memcmp(a, b, n) == 0; };
  const bool odometry = s.n_scans == c.n_scans && s.ring_source == c.ring_source && s.distortion == c.distortion && s.outer_iters == c.outer_iters && s.inner_iters == c.inner_iters &&
                        same(&s.minimum_range, &c.minimum_range, 4) && same(&s.huber, &c.huber, 8) && same(&s.dist_sq_thresh, &c.dist_sq_thresh, 8) &&
                        same(&s.nearby_scan, &c.nearby_scan, 8);
  const bool mapping = s.mapping_skip_frame == c.mapping_skip_frame && same(&s.line_res, &c.line_res, 4) && same(&s.plane_res, &c.plane_res, 4) &&
                       same(s.slab_cap, c.slab_cap, 8) && s.max_map_points == c.max_map_points;
  if (localising(s))
    return odometry && s.mapping_skip_frame == c.mapping_skip_frame && same(&s.line_res, &c.line_res, 4) && same(&s.plane_res, &c.plane_res, 4);
  return odometry && (!s.mapped || mapping);
}

// where a lane's "last" clouds are between two stream calls: the feature slot of the context's latest step
int last_slot(const aloam_ctx* c) { return (c->frame + kFeatSlots - 1) % kFeatSlots; }

// the kind of a caller's snapshot buffer: 1 device memory of this context's device, 0 host memory (pinned or pageable), -1 memory
// the call cannot use (another device, or device memory not aligned to 16 bytes: the store's points are moved as 16-byte words)
int buffer_kind(const aloam_ctx* c, const void* p) { return snapshot_buffer_kind(c, p); }

}  // namespace

bool map_position_fits(const double p[3], const int cen[3]) {
  const int dims[3] = {21, 21, 11};
  for (int a = 0; a < 3; ++a) {
    long long c = 0;
    if (!centre_cube(p[a], cen[a], &c) || c < -kCubeSlack || c >= dims[a] + kCubeSlack) return false;
  }
  return true;
}

int snapshot_buffer_kind(const aloam_ctx* c, const void* p) {
  cudaPointerAttributes at = {};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return -1; }
  if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged)
    return (at.type == cudaMemoryTypeDevice && at.device != c->cfg.device) || reinterpret_cast<uintptr_t>(p) % 16 ? -1 : 1;
  return 0;
}

namespace {

// n bytes between the caller's buffer and host memory, on c->stream (host memory: at once)
int put(aloam_ctx* c, char* dst, bool device, const void* src, size_t n) {
  if (device) CUDA_CHECK_RET(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, c->stream));
  else std::memcpy(dst, src, n);
  return ALOAM_OK;
}
int fetch(aloam_ctx* c, void* dst, const char* src, bool device, size_t n) {
  if (!device) { std::memcpy(dst, src, n); return ALOAM_OK; }
  CUDA_CHECK_RET(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  return ALOAM_OK;
}

int ensure_snap_store(aloam_ctx* c) {
  if (!c->h_snap_store) CUDA_CHECK_RET(halloc(c, &c->h_snap_store, 1));
  return ALOAM_OK;
}

}  // namespace

int snapshot_validate(aloam_ctx* c, const char* b, long long n_bytes, int kind, bool need_mapped, long long* store) {
  if (n_bytes < (long long)sizeof(SnapHeader)) return ALOAM_ERR_SNAPSHOT;
  SnapHeader& h = c->pin->snap;
  int rc = fetch(c, &h, b, kind, sizeof(h)); if (rc) return rc;
  rc = check_header(h, n_bytes); if (rc) return rc;
  if (need_mapped && !h.mapped) return ALOAM_ERR_SNAPSHOT;
  SnapHeader mine = {};
  fingerprint(c, &mine);
  if (!same_config(h, mine)) return ALOAM_ERR_SNAPSHOT;
  *store = store_offset(h);
  if (h.mapped) {
    rc = ensure_snap_store(c); if (rc) return rc;
    rc = fetch(c, c->h_snap_store, b + *store, kind, sizeof(SnapStore)); if (rc) return rc;
    rc = check_store(h, *c->h_snap_store); if (rc) return rc;
  }
  if (localising(h)) {
    rc = fetch(c, &c->pin->snap_loc, b + *store, kind, sizeof(SnapLocalise)); if (rc) return rc;
    rc = check_localise(h, c->pin->snap_loc); if (rc) return rc;
  }
  return ALOAM_OK;
}

namespace {

// the host checks of a snapshot in host memory, without a context: *h its header, *loc its locator section (format 2)
int check_host_blob(const void* blob, long long n_bytes, SnapHeader* h, SnapStore* store, SnapLocalise* loc) {
  if (n_bytes < (long long)sizeof(SnapHeader)) return ALOAM_ERR_SNAPSHOT;
  const char* b = static_cast<const char*>(blob);
  std::memcpy(h, b, sizeof(*h));
  int rc = check_header(*h, n_bytes); if (rc) return rc;
  if (h->mapped) {
    std::memcpy(store, b + store_offset(*h), sizeof(SnapStore));   // (the blob need not be aligned)
    rc = check_store(*h, *store); if (rc) return rc;
  }
  if (localising(*h)) {
    std::memcpy(loc, b + store_offset(*h), sizeof(SnapLocalise));
    rc = check_localise(*h, *loc); if (rc) return rc;
  }
  return ALOAM_OK;
}

// aloam_lane_save (format 1) and aloam_lane_save_localising (format 2, `loc`) of a lane whose mode the caller has checked
int save_lane(aloam_ctx* c, int lane, void* out, long long capacity, long long* n_bytes, bool loc) {
  const Lane& L = c->lanes[lane];
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const FeatBuf& f = L.feat[last_slot(c)];
  SnapHeader& h = c->pin->snap;
  std::memset(&h, 0, sizeof(h));
  SnapLocalise& s = c->pin->snap_loc;
  if (loc) std::memset(&s, 0, sizeof(s));
  CUDA_CHECK_RET(cudaMemcpyAsync(c->pin->snap_counts, f.counts, 16, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(h.warm, L.d_pose, 56, cudaMemcpyDeviceToHost, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(h.world, L.d_world, 56, cudaMemcpyDeviceToHost, c->stream));
  double T[7];
  if (loc) { int rc = locator_map_pose(c, lane, T); if (rc) return rc; }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  std::memcpy(h.magic, kMagic, 8);
  h.version = loc ? kSnapVersionLocalise : kSnapVersion;
  h.mapped = loc ? 0 : L.sched.mapped;
  h.scan_index = L.sched.scan;
  h.n_less_sharp = c->pin->snap_counts[1];
  h.n_less_flat = c->pin->snap_counts[3];
  fingerprint(c, &h);
  const long long store = store_offset(h);
  h.total_bytes = store;
  int rc = ALOAM_OK;
  if (h.mapped) {
    rc = ensure_snap_store(c); if (rc) return rc;
    rc = mapper_store_tables(c, lane, c->h_snap_store, &h.cube_growth); if (rc) return rc;   // the lane's own, not the context's
    h.total_bytes += (long long)sizeof(SnapStore) + 16 * c->h_snap_store->n_points;
  }
  if (loc) {   // T_wmap_wodom after the lane's last frame (and any recovery it adopted), and the map it localises against
    for (int k = 0; k < 4; ++k) s.q_wmap_wodom[k] = T[k];
    for (int k = 0; k < 3; ++k) s.t_wmap_wodom[k] = T[4 + k];
    long long n[2];
    unsigned long long digest = 0;
    rc = prior_map_identity(c, s.centre, n, &digest); if (rc) return rc;
    s.digest = digest;
    s.map_points[0] = n[0]; s.map_points[1] = n[1];
    h.total_bytes += (long long)sizeof(SnapLocalise);
  }
  *n_bytes = h.total_bytes;
  if (!out && capacity == 0) return ALOAM_OK;   // the size only
  if (!out) return ALOAM_ERR_INVALID_ARG;
  if (capacity < h.total_bytes) return ALOAM_ERR_CAPACITY;
  const int kind = buffer_kind(c, out);
  if (kind < 0) return ALOAM_ERR_INVALID_ARG;
  char* o = static_cast<char*>(out);
  rc = put(c, o, kind, &h, sizeof(h)); if (rc) return rc;
  if (h.n_less_sharp > 0) CUDA_CHECK_RET(cudaMemcpyAsync(o + sizeof(h), f.less_sharp, 16 * (size_t)h.n_less_sharp, cudaMemcpyDefault, c->stream));
  if (h.n_less_flat > 0) CUDA_CHECK_RET(cudaMemcpyAsync(o + sizeof(h) + 16 * (size_t)h.n_less_sharp, f.less_flat, 16 * (size_t)h.n_less_flat, cudaMemcpyDefault, c->stream));
  if (h.mapped) {
    rc = put(c, o + store, kind, c->h_snap_store, sizeof(SnapStore)); if (rc) return rc;
    rc = mapper_store_points(c, lane, c->h_snap_store->n_points, o + store + sizeof(SnapStore), kind); if (rc) return rc;
  }
  if (loc) { rc = put(c, o + store, kind, &s, sizeof(s)); if (rc) return rc; }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  return ALOAM_OK;
}

}  // namespace

extern "C" {

int aloam_snapshot_check(const void* blob, long long n_bytes, aloam_snapshot_info* info) {
  if (!blob || n_bytes < 0) return ALOAM_ERR_INVALID_ARG;
  SnapHeader h;
  std::vector<char> buf(sizeof(SnapStore));
  SnapStore* s = reinterpret_cast<SnapStore*>(buf.data());
  SnapLocalise loc;
  const int rc = check_host_blob(blob, n_bytes, &h, s, &loc); if (rc) return rc;
  if (info) {
    info->version = h.version; info->mapped = h.mapped; info->n_scans = h.n_scans; info->scan_index = h.scan_index;
    info->bytes = h.total_bytes; info->map_points = h.mapped ? s->n_points : 0;
    for (int k = 0; k < 7; ++k) info->world[k] = h.world[k];
  }
  return ALOAM_OK;
}

int aloam_snapshot_localise_info(const void* blob, long long n_bytes, double t_wmap_wodom[7], unsigned long long* digest, int centre[3],
                                 long long map_points[2]) {
  if (!blob || n_bytes < 0) return ALOAM_ERR_INVALID_ARG;
  SnapHeader h;
  std::vector<char> buf(sizeof(SnapStore));
  SnapLocalise loc;
  const int rc = check_host_blob(blob, n_bytes, &h, reinterpret_cast<SnapStore*>(buf.data()), &loc); if (rc) return rc;
  if (!localising(h)) return ALOAM_ERR_SNAPSHOT;
  if (t_wmap_wodom) {
    for (int k = 0; k < 4; ++k) t_wmap_wodom[k] = loc.q_wmap_wodom[k];
    for (int k = 0; k < 3; ++k) t_wmap_wodom[4 + k] = loc.t_wmap_wodom[k];
  }
  if (digest) *digest = loc.digest;
  if (centre) for (int a = 0; a < 3; ++a) centre[a] = loc.centre[a];
  if (map_points) for (int t = 0; t < 2; ++t) map_points[t] = loc.map_points[t];
  return ALOAM_OK;
}

int aloam_lane_save(aloam_ctx* c, int lane, void* out, long long capacity, long long* n_bytes) {
  if (!c || !n_bytes || capacity < 0 || lane < 0 || lane >= c->n_lanes) return ALOAM_ERR_INVALID_ARG;
  const Lane& L = c->lanes[lane];
  if (!c->lanes_mode || !L.sched.running) return ALOAM_ERR_STATE;
  if (L.sched.localising) return ALOAM_ERR_STATE;   // format 1 has no section for a localising lane: aloam_lane_save_localising
  return save_lane(c, lane, out, capacity, n_bytes, false);
}

int aloam_lane_save_localising(aloam_ctx* c, int lane, void* out, long long capacity, long long* n_bytes) {
  if (!c || !n_bytes || capacity < 0 || lane < 0 || lane >= c->n_lanes) return ALOAM_ERR_INVALID_ARG;
  const Lane& L = c->lanes[lane];
  if (!c->lanes_mode || !L.sched.running || !L.sched.localising || !L.locator || !c->prior) return ALOAM_ERR_STATE;
  return save_lane(c, lane, out, capacity, n_bytes, true);
}

int aloam_lane_restore(aloam_ctx* c, int lane, const void* blob, long long n_bytes) {
  if (!c || !blob || n_bytes < 0 || lane < 0 || lane >= c->n_lanes) return ALOAM_ERR_INVALID_ARG;
  if (sharded_job(c)) return ALOAM_ERR_STATE;   // as aloam_scan_stream_lanes
  CUDA_CHECK_RET(cudaSetDevice(c->cfg.device));
  const int kind = buffer_kind(c, blob);
  if (kind < 0) return ALOAM_ERR_INVALID_ARG;
  // as at a START: the lane's trajectory, if any, ends here, and the context runs lanes from now on
  Lane& L = c->lanes[lane];
  c->lanes_mode = true;
  L.sched.running = L.sched.localising = false;
  if (const int rc = place_clear(c, lane)) return rc;   // keyframes are not part of snapshots
  // ---- validation, on the host, before anything is written to the device
  const char* b = static_cast<const char*>(blob);
  const SnapHeader& h = c->pin->snap;
  long long store = 0;
  int rc = snapshot_validate(c, b, n_bytes, kind, false, &store); if (rc) return rc;
  if (h.n_less_sharp > c->max_points || h.n_less_flat > c->max_points) return ALOAM_ERR_CAPACITY;
  const bool loc = localising(h);
  double T[7];
  if (loc) {   // the lane localises against the context's prior map: it must be the map the snapshot names
    if (!c->prior) return ALOAM_ERR_STATE;
    if (c->cfg.max_map_points <= 0) return ALOAM_ERR_SNAPSHOT;   // no mapped stream call could continue it
    const SnapLocalise& s = c->pin->snap_loc;
    int cen[3];
    long long n[2];
    unsigned long long digest = 0;
    rc = prior_map_identity(c, cen, n, &digest); if (rc) return rc;
    for (int a = 0; a < 3; ++a) if (cen[a] != s.centre[a]) return ALOAM_ERR_SNAPSHOT;
    if (n[0] != s.map_points[0] || n[1] != s.map_points[1] || digest != s.digest) return ALOAM_ERR_SNAPSHOT;
    for (int k = 0; k < 4; ++k) T[k] = s.q_wmap_wodom[k];
    for (int k = 0; k < 3; ++k) T[4 + k] = s.t_wmap_wodom[k];
    rc = locator_ensure(c, lane); if (rc) return rc;
  }
  for (int l = 0; h.mapped && l <= lane; ++l) { rc = mapper_ensure(c, l); if (rc) return rc; }   // the stores of lanes 0 .. lane, if needed
  // ---- odometry: the "last" clouds into the slot the next step reads, their index and ring check, the poses, the armed scalars
  const int slot = last_slot(c);
  FeatBuf& f = L.feat[slot];
  if (h.n_less_sharp > 0) CUDA_CHECK_RET(cudaMemcpyAsync(f.less_sharp, b + sizeof(h), 16 * (size_t)h.n_less_sharp, cudaMemcpyDefault, c->stream));
  if (h.n_less_flat > 0) CUDA_CHECK_RET(cudaMemcpyAsync(f.less_flat, b + sizeof(h) + 16 * (size_t)h.n_less_sharp, 16 * (size_t)h.n_less_flat, cudaMemcpyDefault, c->stream));
  int* lc = c->pin->snap_counts;
  lc[0] = 0; lc[1] = h.n_less_sharp; lc[2] = 0; lc[3] = h.n_less_flat;
  CUDA_CHECK_RET(cudaMemcpyAsync(f.counts, lc, 16, cudaMemcpyHostToDevice, c->stream));
  rc = index_last_clouds(c, lane, slot, h.n_less_sharp, h.n_less_flat); if (rc) return rc;
  CUDA_CHECK_RET(cudaMemcpyAsync(L.d_pose, h.warm, 56, cudaMemcpyHostToDevice, c->stream));
  CUDA_CHECK_RET(cudaMemcpyAsync(L.d_world, h.world, 56, cudaMemcpyHostToDevice, c->stream));
  // k_ring_scan arms a lane's next ScanScalars slot only when the lane ran the step before
  CUDA_CHECK_RET(cudaMemcpyAsync(L.d_sc + c->parity, c->d_sc_init, sizeof(ScanScalars), cudaMemcpyDeviceToDevice, c->stream));
  // ---- the cube store, or the locator's frame state
  if (h.mapped) { rc = mapper_store_restore(c, lane, c->h_snap_store, b + store + sizeof(SnapStore), kind, h.cube_growth != 0); if (rc) return rc; }
  if (loc) { rc = locator_restore(c, lane, T); if (rc) return rc; }
  CUDA_CHECK_RET(cudaStreamSynchronize(c->stream));
  CUDA_CHECK_RET(cudaGetLastError());
  L.sched.running = true;
  L.sched.mapped = h.mapped != 0 || loc;
  L.sched.localising = loc;
  L.sched.scan = h.scan_index;
  if (loc) L.window = false;   // no frame of this trajectory has run in this context yet
  return ALOAM_OK;
}

}  // extern "C"
