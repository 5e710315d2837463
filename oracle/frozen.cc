// ORACLE (test infrastructure) -- the frozen-map frame behind localisation against a prior map, as a flat C interface for ctypes
// (oracle/pyfrozen.py).  Built into oracle/libfrozen.so by `make -C oracle -f frozen.mk libfrozen.so`.
//
// A frozen frame is alaserMapping's frame (laserMapping.cpp:309-734) with two parts left out:
//   * no ring-buffer shift (:323-507): the centre offsets are those of the prior map; centerCubeI/J/K as at :312-321, and the
//     5 x 5 x 3 window of :512-531 clipped to the buffer by that loop's own bounds test, in its order;
//   * no insertion and no re-filter (:736-801): the store is never written.
// Pose hand-off (transformAssociateToMap), the stack filters, the thin-map test of :554, association + the two solves through
// orc::Mapping, and transformUpdate are the ordinary frame's (oracle/cubemap.cc), so a frozen frame and CubeMap::step started from
// the same store and T_wmap_wodom return the same pose bit for bit while the latter would not shift.
#include <cmath>
#include "oracle.h"

namespace {
constexpr int W = 21, H = 21, D = 11;
inline int cube_index(int i, int j, int k) { return i + W * j + W * H * k; }
inline int cube_coord(double v, int centre) {   // :314-325
  int c = int((v + 25.0) / 50.0) + centre;
  if (v + 25.0 < 0) c--;
  return c;
}

struct FrozenMap {
  std::vector<orc::Cloud> corner, surf;   // the prior map's cubes: never written by a frame
  int cen[3] = {10, 10, 5};
  FrozenMap() : corner(W * H * D), surf(W * H * D) {}
};
}  // namespace

extern "C" {

void* orc_frozen_create(const int cen[3]) {
  FrozenMap* m = new FrozenMap();
  for (int a = 0; a < 3; ++a) m->cen[a] = cen[a];
  return m;
}
void orc_frozen_free(void* h) { delete (FrozenMap*)h; }
int orc_frozen_set_cube(void* h, int which, int index, const float* pts, int n) {
  FrozenMap* m = (FrozenMap*)h;
  if (index < 0 || index >= W * H * D) return -1;
  orc::Cloud& c = which == 0 ? m->corner[index] : m->surf[index];
  c.resize(n);
  for (int i = 0; i < n; ++i) c[i] = orc::PointXYZI{pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]};
  return 0;
}
int orc_frozen_get_cube(void* h, int which, int index, float* out, int cap) {
  FrozenMap* m = (FrozenMap*)h;
  if (index < 0 || index >= W * H * D) return -1;
  const orc::Cloud& c = which == 0 ? m->corner[index] : m->surf[index];
  const int n = (int)c.size();
  for (int i = 0; i < n && i < cap; ++i) { out[4 * i] = c[i].x; out[4 * i + 1] = c[i].y; out[4 * i + 2] = c[i].z; out[4 * i + 3] = c[i].intensity; }
  return n;
}

// one frozen frame of a lane whose map-to-odometry transform is (q_wmap_wodom, t_wmap_wodom), updated in place (transformUpdate).
// pose7 = parameters[7] afterwards; valid = the clipped window in loop order; info = {optimised, n valid, corner / surf points of
// the window, corner / surf stack sizes}.  Returns 1 when the optimisation ran.
int orc_frozen_step(void* h, const float* corner, int nc, const float* surf, int ns, const double q_odom[4], const double t_odom[3],
                    double q_wmap_wodom[4], double t_wmap_wodom[3], float line_res, float plane_res, int outer, int max_iters, int sort_mode,
                    double pose7[7], int valid[75], int info[6]) {
  const FrozenMap* m = (const FrozenMap*)h;
  orc::SolveOptions opt; opt.max_num_iterations = max_iters;
  orc::Cloud c(nc), s(ns);
  for (int i = 0; i < nc; ++i) c[i] = orc::PointXYZI{corner[4 * i], corner[4 * i + 1], corner[4 * i + 2], corner[4 * i + 3]};
  for (int i = 0; i < ns; ++i) s[i] = orc::PointXYZI{surf[4 * i], surf[4 * i + 1], surf[4 * i + 2], surf[4 * i + 3]};
  double x[7];
  orc::transform_associate_to_map(q_wmap_wodom, t_wmap_wodom, q_odom, t_odom, x);   // :311
  const int ci = cube_coord(x[4], m->cen[0]), cj = cube_coord(x[5], m->cen[1]), ck = cube_coord(x[6], m->cen[2]);   // :314-325, no shift
  int nv = 0;
  orc::Cloud corner_from_map, surf_from_map;
  for (int i = ci - 2; i <= ci + 2; ++i)
    for (int j = cj - 2; j <= cj + 2; ++j)
      for (int k = ck - 1; k <= ck + 1; ++k)
        if (i >= 0 && i < W && j >= 0 && j < H && k >= 0 && k < D) {   // :512-539
          const int ind = cube_index(i, j, k);
          valid[nv++] = ind;
          corner_from_map.insert(corner_from_map.end(), m->corner[ind].begin(), m->corner[ind].end());
          surf_from_map.insert(surf_from_map.end(), m->surf[ind].begin(), m->surf[ind].end());
        }
  orc::Cloud corner_stack, surf_stack;
  orc::voxel_grid(c, line_res, (orc::SortMode)sort_mode, corner_stack);   // :541-550
  orc::voxel_grid(s, plane_res, (orc::SortMode)sort_mode, surf_stack);
  orc::Mapping reg;
  reg.set_map(corner_from_map, surf_from_map);
  const int optimised = reg.register_scan(corner_stack, surf_stack, x, outer, opt);   // :554-733
  orc::transform_update(x, q_odom, t_odom, q_wmap_wodom, t_wmap_wodom);               // :734
  for (int k = 0; k < 7; ++k) pose7[k] = x[k];
  info[0] = optimised; info[1] = nv; info[2] = (int)corner_from_map.size(); info[3] = (int)surf_from_map.size();
  info[4] = (int)corner_stack.size(); info[5] = (int)surf_stack.size();
  return optimised;
}

// the high-frequency pose of a scan the lane does not register (laserMapping.cpp:197-229): T_wmap_wodom * odometry pose
void orc_frozen_high_freq(const double q_wmap_wodom[4], const double t_wmap_wodom[3], const double q_odom[4], const double t_odom[3], double pose7[7]) {
  orc::transform_associate_to_map(q_wmap_wodom, t_wmap_wodom, q_odom, t_odom, pose7);
}

}  // extern "C"
