// Internal: lane snapshot formats v1 (aloam_lane_save / aloam_lane_restore / aloam_snapshot_check) and v2 (a localising lane:
// aloam_lane_save_localising), shared by snapshot.cu and cubemap.cu.  include/aloam_b200.h documents the same layouts for callers:
// little-endian, every section 16-byte aligned.
#pragma once
#include <cstddef>
#include <cstdint>

namespace aloam {

constexpr int kSnapVersion = 1;
constexpr int kSnapVersionLocalise = 2;   // the v1 header (mapped 0, cube_growth 0), the "last" clouds, then SnapLocalise
constexpr int kSnapCubes = 4851;   // 21 x 21 x 11 cubes of the mapper's ring buffer
constexpr int kSnapValid = 128;
constexpr int kSnapPool = 1024;    // slabs per cloud type: the runs of a type's cubes take at most this many

// section 1, at offset 0
struct SnapHeader {
  char magic[8];                       // "ALOAMLS1"
  int32_t version, mapped;
  int64_t total_bytes;
  int32_t scan_index;                  // index of the lane's next scan in its trajectory (mapping_skip_frame)
  int32_t n_less_sharp, n_less_flat;   // the "last" clouds of section 2
  // the configuration the snapshot was taken under: every field that can change a result
  int32_t n_scans, distortion, mapping_skip_frame, outer_iters, inner_iters;
  float minimum_range, line_res, plane_res;
  int32_t slab_cap[2];                 // points per slab: min(16384, max_points), min(65536, max_points)
  int32_t max_map_points;
  double huber, dist_sq_thresh, nearby_scan;
  double warm[7];                      // para_q / para_t of the next scan's solve
  double world[7];                     // world pose of the lane's last scan
  int32_t ring_source;                 // 0 elevation (what a snapshot written before the field held), 1 driver ring
  int32_t cube_growth;                 // the store's cube growth: 0 off (what a snapshot written before the field held), 1 on
  char zero[32];
};
static_assert(sizeof(SnapHeader) == 256, "snapshot header");
static_assert(offsetof(SnapHeader, scan_index) == 24 && offsetof(SnapHeader, n_scans) == 36 && offsetof(SnapHeader, minimum_range) == 56 &&
              offsetof(SnapHeader, slab_cap) == 68 && offsetof(SnapHeader, huber) == 80 && offsetof(SnapHeader, warm) == 104 &&
              offsetof(SnapHeader, world) == 160 && offsetof(SnapHeader, ring_source) == 216 &&
              offsetof(SnapHeader, cube_growth) == 220, "snapshot header layout");

// section 2 at offset 256: n_less_sharp, then n_less_flat points of 4 floats.  Section 3 (mapped snapshots only) follows: this
// table, then n_points points of 4 floats in ALOAM_EXPORT_MAP order
struct SnapStore {
  int32_t cen[3], n_valid;
  int32_t valid[kSnapValid];          // entries n_valid .. 127 are 0
  int32_t frames, zero0;
  double q_wmap_wodom[4], t_wmap_wodom[3];
  int32_t count[2][kSnapCubes];       // points of cube i of type t (0 corner, 1 surf); -1: the cube holds no run
  int32_t zero1[2];
  int64_t n_points;
  int64_t zero2;
};
static_assert(sizeof(SnapStore) == 39424, "snapshot store table");
static_assert(offsetof(SnapStore, frames) == 528 && offsetof(SnapStore, q_wmap_wodom) == 536 && offsetof(SnapStore, count) == 592 &&
              offsetof(SnapStore, n_points) == 39408, "snapshot store table layout");

// section 3 of a format-2 snapshot (a localising lane), at S = 256 + 16 (n_less_sharp + n_less_flat): the lane's T_wmap_wodom
// and what names the prior map it localises against
struct SnapLocalise {
  double q_wmap_wodom[4], t_wmap_wodom[3];
  uint64_t digest;                     // aloam_prior_map_digest of the map
  int32_t centre[3], zero0;            // its centre offsets
  int64_t map_points[2];               // its corner / surf points
  char zero1[32];
};
static_assert(sizeof(SnapLocalise) == 128, "localising snapshot section");
static_assert(offsetof(SnapLocalise, t_wmap_wodom) == 32 && offsetof(SnapLocalise, digest) == 56 && offsetof(SnapLocalise, centre) == 64 &&
              offsetof(SnapLocalise, map_points) == 80, "localising snapshot section layout");

}  // namespace aloam
