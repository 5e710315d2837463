// Eigen-order quaternion helpers (the operation order of Eigen::Quaternion), shared by the mapper's pose hand-off (cubemap.cu) and
// the recovery candidates (recover.cu): both are compared bit for bit with host transcriptions, so every caller is compiled
// -fmad=false.
#pragma once

namespace aloam {

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

}  // namespace aloam
