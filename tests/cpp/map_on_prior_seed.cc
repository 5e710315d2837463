// TEST INFRASTRUCTURE (tests/map_on_prior_seed.py compiles it at test time): the starting state of a mapping trajectory on a copy
// of a prior map (aloam_lane_map_on_prior), written into the two CPU mappers the device is checked against.
//   - seed_cubemap: the public state of an oracle orc::CubeMap (liboracle.so's orc_cubemap_create handle);
//   - seed_ref_node: the file-scope globals of the reference's own laserMapping.cpp inside a loaded oracle/_ref/libref_mapping.so,
//     passed in by address: laserCloudCornerArray / laserCloudSurfArray, laserCloudCen*, q_wmap_wodom, t_wmap_wodom.  Only the
//     stand-in headers of oracle/ref_shim are compiled here (the types of those globals), no reference source.
// Both take the store as counts[2][4851] (points of corner / surf cube i, < 0 = none) and the points in ALOAM_EXPORT_MAP order
// (corner cube i, then surf cube i, for i = 0 .. 4850; 4 floats each).
#include "oracle.h"
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#include <eigen3/Eigen/Dense>

namespace {
constexpr int kCubes = 21 * 21 * 11;
inline int count_of(const int* counts, int ty, int i) { const int n = counts[ty * kCubes + i]; return n > 0 ? n : 0; }
}  // namespace

extern "C" {

// centre offsets cen, T_wmap_wodom (q xyzw, t), every cube; no valid list, frames = 0
void seed_cubemap(void* h, const int cen[3], const double q[4], const double t[3], const int* counts, const float* pts) {
  orc::CubeMap* m = static_cast<orc::CubeMap*>(h);
  m->cen_w = cen[0]; m->cen_h = cen[1]; m->cen_d = cen[2];
  for (int k = 0; k < 4; ++k) m->q_wmap_wodom[k] = q[k];
  for (int k = 0; k < 3; ++k) m->t_wmap_wodom[k] = t[k];
  long long off = 0;
  for (int i = 0; i < kCubes; ++i)
    for (int ty = 0; ty < 2; ++ty) {
      orc::Cloud& c = ty ? m->surf[i] : m->corner[i];
      c.resize(count_of(counts, ty, i));
      for (orc::PointXYZI& p : c) { p = orc::PointXYZI{pts[4 * off], pts[4 * off + 1], pts[4 * off + 2], pts[4 * off + 3]}; ++off; }
    }
  m->valid.clear();
  m->frames = 0;
}

// after ref_map_init, before the node's first frame
void seed_ref_node(void* corner_array, void* surf_array, int* cen_w, int* cen_h, int* cen_d, void* q_wmap_wodom, void* t_wmap_wodom,
                   const int cen[3], const double q[4], const double t[3], const int* counts, const float* pts) {
  typedef pcl::PointCloud<pcl::PointXYZI>::Ptr CloudPtr;
  CloudPtr* arrays[2] = {static_cast<CloudPtr*>(corner_array), static_cast<CloudPtr*>(surf_array)};
  *cen_w = cen[0]; *cen_h = cen[1]; *cen_d = cen[2];
  *static_cast<Eigen::Quaterniond*>(q_wmap_wodom) = Eigen::Quaterniond(q[3], q[0], q[1], q[2]);
  *static_cast<Eigen::Vector3d*>(t_wmap_wodom) = Eigen::Vector3d(t[0], t[1], t[2]);
  long long off = 0;
  for (int i = 0; i < kCubes; ++i)
    for (int ty = 0; ty < 2; ++ty) {
      pcl::PointCloud<pcl::PointXYZI>& c = *arrays[ty][i];
      c.clear();
      for (int j = count_of(counts, ty, i); j > 0; --j, ++off) {
        pcl::PointXYZI p;
        p.x = pts[4 * off]; p.y = pts[4 * off + 1]; p.z = pts[4 * off + 2]; p.intensity = pts[4 * off + 3];
        c.push_back(p);
      }
    }
}

}  // extern "C"
