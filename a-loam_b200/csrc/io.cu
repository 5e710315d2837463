// Host-side format helpers (include/aloam_io.h): KITTI .bin scans and pose files, PointCloud2 payloads of
// pcl::PointXYZI.  No device code; the file has a .cu suffix only because the library is built from one source list.
// Follows kittiHelper.cpp:25-35 (file read), :78-80 and :97-113 (pose parsing through float, camera -> lidar frame).
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include "../../include/aloam_io.h"

namespace {

struct Q { double x, y, z, w; };

// Eigen::Quaterniond(Matrix3d) -- Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl<Other, 3, 3>
Q quat_from_matrix(const double m[3][3]) {
  Q q;
  double t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0.0) {
    t = std::sqrt(t + 1.0);
    q.w = 0.5 * t;
    t = 0.5 / t;
    q.x = (m[2][1] - m[1][2]) * t;
    q.y = (m[0][2] - m[2][0]) * t;
    q.z = (m[1][0] - m[0][1]) * t;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    double v[3];
    v[i] = 0.5 * t;
    t = 0.5 / t;
    q.w = (m[k][j] - m[j][k]) * t;
    v[j] = (m[j][i] + m[i][j]) * t;
    v[k] = (m[k][i] + m[i][k]) * t;
    q.x = v[0]; q.y = v[1]; q.z = v[2];
  }
  return q;
}

Q qmul(const Q& a, const Q& b) {  // Eigen quaternion product
  return Q{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
           a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}

void qrot(const Q& q, const double v[3], double o[3]) {  // Eigen: v + w*uv + u x uv with uv = 2 u x v
  const double ux = q.x, uy = q.y, uz = q.z;
  double uvx = uy * v[2] - uz * v[1], uvy = uz * v[0] - ux * v[2], uvz = ux * v[1] - uy * v[0];
  uvx += uvx; uvy += uvy; uvz += uvz;
  o[0] = v[0] + q.w * uvx + (uy * uvz - uz * uvy);
  o[1] = v[1] + q.w * uvy + (uz * uvx - ux * uvz);
  o[2] = v[2] + q.w * uvz + (ux * uvy - uy * uvx);
}

void qmat(const Q& q, double m[3][3]) {
  const double x = q.x, y = q.y, z = q.z, w = q.w;
  m[0][0] = 1 - 2 * (y * y + z * z); m[0][1] = 2 * (x * y - z * w); m[0][2] = 2 * (x * z + y * w);
  m[1][0] = 2 * (x * y + z * w); m[1][1] = 1 - 2 * (x * x + z * z); m[1][2] = 2 * (y * z - x * w);
  m[2][0] = 2 * (x * z - y * w); m[2][1] = 2 * (y * z + x * w); m[2][2] = 1 - 2 * (x * x + y * y);
}

const double kRt[3][3] = {{0, 0, 1}, {-1, 0, 0}, {0, -1, 0}};  // kittiHelper.cpp:78-79

}  // namespace

extern "C" {

long aloam_io_kitti_bin_points(const char* path) {
  FILE* f = path ? std::fopen(path, "rb") : nullptr;
  if (!f) return -1;
  std::fseek(f, 0, SEEK_END);
  const long bytes = std::ftell(f);
  std::fclose(f);
  return bytes < 0 ? -1 : (long)((size_t)bytes / sizeof(float)) / 4;
}

long aloam_io_read_kitti_bin(const char* path, float* xyzi, long capacity_points) {
  if (!xyzi || capacity_points < 0) return -1;
  FILE* f = path ? std::fopen(path, "rb") : nullptr;
  if (!f) return -1;
  const size_t got = std::fread(xyzi, 4 * sizeof(float), (size_t)capacity_points, f);
  std::fclose(f);
  return (long)got;
}

int aloam_io_parse_kitti_pose(const char* line, double T[12]) {
  if (!line || !T) return -1;
  const char* p = line;
  for (int i = 0; i < 12; ++i) {
    char* end = nullptr;
    const float v = std::strtof(p, &end);   // stof(): the reference reads the ground truth through float
    if (end == p) return -1;
    T[i] = (double)v;
    p = end;
  }
  return 0;
}

void aloam_io_kitti_pose_to_lidar(const double T[12], double q[4], double t[3]) {
  double R[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[i][j] = T[4 * i + j];
  const Q qt = quat_from_matrix(kRt);
  Q r = qmul(qt, quat_from_matrix(R));
  const double n = std::sqrt(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
  r.x /= n; r.y /= n; r.z /= n; r.w /= n;
  q[0] = r.x; q[1] = r.y; q[2] = r.z; q[3] = r.w;
  const double tc[3] = {T[3], T[7], T[11]};
  qrot(qt, tc, t);
}

void aloam_io_lidar_pose_to_kitti(const double q[4], const double t[3], double T[12]) {
  // R_cam = Rt^T R_lidar, t_cam = Rt^T t_lidar
  double Rl[3][3];
  qmat(Q{q[0], q[1], q[2], q[3]}, Rl);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += kRt[k][i] * Rl[k][j];
      T[4 * i + j] = s;
    }
    T[4 * i + 3] = kRt[0][i] * t[0] + kRt[1][i] * t[1] + kRt[2][i] * t[2];
  }
}

void aloam_io_pack_pointxyzi(const float* xyzi, long n, unsigned char* data32) {
  for (long i = 0; i < n; ++i) {
    unsigned char* o = data32 + 32 * i;
    std::memset(o, 0, 32);
    std::memcpy(o, xyzi + 4 * i, 12);             // x, y, z ; bytes 12..15: the SSE padding of PCL_ADD_POINT4D
    std::memcpy(o + 16, xyzi + 4 * i + 3, 4);     // intensity
  }
}

int aloam_io_unpack_points(const unsigned char* data, long n, int point_step, int off_x, int off_y, int off_z,
                           int off_intensity, float* xyzi) {
  if (!data || !xyzi || n < 0 || point_step < 12 || off_x < 0 || off_y < 0 || off_z < 0) return -1;
  if (off_x + 4 > point_step || off_y + 4 > point_step || off_z + 4 > point_step || off_intensity + 4 > point_step) return -1;
  for (long i = 0; i < n; ++i) {
    const unsigned char* p = data + (size_t)point_step * i;
    std::memcpy(xyzi + 4 * i, p + off_x, 4);
    std::memcpy(xyzi + 4 * i + 1, p + off_y, 4);
    std::memcpy(xyzi + 4 * i + 2, p + off_z, 4);
    if (off_intensity >= 0) std::memcpy(xyzi + 4 * i + 3, p + off_intensity, 4);
    else xyzi[4 * i + 3] = 0.f;
  }
  return 0;
}

int aloam_io_unpack_points_ring(const unsigned char* data, long n, int point_step, int off_x, int off_y, int off_z, int off_ring,
                                int ring_type, float* xyzr) {
  const int ring_bytes = ring_type == 2 ? 1 : ring_type == 4 ? 2 : 0;   // sensor_msgs/PointField UINT8, UINT16
  if (!data || !xyzr || n < 0 || ring_bytes == 0 || point_step < 12 || off_x < 0 || off_y < 0 || off_z < 0 || off_ring < 0) return -1;
  if (off_x + 4 > point_step || off_y + 4 > point_step || off_z + 4 > point_step || off_ring + ring_bytes > point_step) return -1;
  for (long i = 0; i < n; ++i) {
    const unsigned char* p = data + (size_t)point_step * i;
    std::memcpy(xyzr + 4 * i, p + off_x, 4);
    std::memcpy(xyzr + 4 * i + 1, p + off_y, 4);
    std::memcpy(xyzr + 4 * i + 2, p + off_z, 4);
    uint16_t r = p[off_ring];
    if (ring_bytes == 2) std::memcpy(&r, p + off_ring, 2);   // little-endian payload (is_bigendian = false)
    xyzr[4 * i + 3] = (float)r;
  }
  return 0;
}

}  // extern "C"
