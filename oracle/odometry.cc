// ORACLE (test infrastructure) -- scan-to-scan registration of laserOdometry.cpp:
//   :111-129  TransformToStart (DISTORTION 0 => s = 1, DISTORTION 1 => per-point ratio; double math, rounded to float on store)
//   :278-501  2 x { corner association (:299-384), plane association (:387-483), ceres::Solve (:494-499) }
//   :504-505  pose integration            :554-568  swap "last" clouds, rebuild both kd-trees
// All squared distances in the ring-window scans are float expressions (operands are float members; only the
// result is widened to double, :322-327) and the break tests compare int ring ids with a double (+-NEARBY_SCAN).
#include <cmath>
#include "oracle.h"

namespace orc {

namespace {
const double SCAN_PERIOD = 0.1;           // :64

// interpolation ratio (:113-118,376-379): float intensity minus its integer part (float arithmetic), divided by the double
inline double ratio_of(const PointXYZI& pi, bool distortion) {
  if (distortion) return (pi.intensity - int(pi.intensity)) / SCAN_PERIOD;
  return 1.0;
}

// :111-129
inline PointXYZI transform_to_start(const PointXYZI& pi, const Quat& q_last_curr, const Vec3& t_last_curr, bool distortion) {
  const double s = ratio_of(pi, distortion);
  Quat q_point_last = slerp(Quat{0, 0, 0, 1}, s, q_last_curr);
  Vec3 t_point_last{s * t_last_curr.x, s * t_last_curr.y, s * t_last_curr.z};
  Vec3 point{pi.x, pi.y, pi.z};
  Vec3 un_point = rotate(q_point_last, point) + t_point_last;
  PointXYZI po;
  po.x = (float)un_point.x; po.y = (float)un_point.y; po.z = (float)un_point.z;
  po.intensity = pi.intensity;
  return po;
}
inline float sqdist_f(const PointXYZI& a, const PointXYZI& b) {
  return (a.x - b.x) * (a.x - b.x) + (a.y - b.y) * (a.y - b.y) + (a.z - b.z) * (a.z - b.z);
}
inline int ring(const PointXYZI& p) { return int(p.intensity); }
}  // namespace

void Odometry::set_last(const Cloud& c, const Cloud& s) {
  double t0 = now_ms();
  corner_last = c;
  surf_last = s;
  tree_corner.build(corner_last);
  tree_surf.build(surf_last);
  times.tree_ms = now_ms() - t0;
}

void Odometry::associate(const Cloud& sharp, const Cloud& flat, const double qv[4], const double tv[3],
                         std::vector<Correspondence>* ccorr, std::vector<Correspondence>* pcorr,
                         std::vector<ResidualBlock>* blocks) const {
  const double DISTANCE_SQ_THRESHOLD = dist_sq_thresh;   // laserOdometry.cpp:65 (25 there)
  const double NEARBY_SCAN = nearby_scan;                // :66 (2.5 there)
  const Quat q{qv[0], qv[1], qv[2], qv[3]};
  const Vec3 t{tv[0], tv[1], tv[2]};
  const int n_corner_last = (int)corner_last.size(), n_surf_last = (int)surf_last.size();
  int nn_idx; float nn_d;

  for (int i = 0; i < (int)sharp.size(); ++i) {  // :299
    PointXYZI sel = transform_to_start(sharp[i], q, t, distortion);
    const float qq[3] = {sel.x, sel.y, sel.z};
    if (tree_corner.knn(qq, 1, &nn_idx, &nn_d) < 1) continue;  // (PCL would return 0 neighbours on an empty tree)
    int closest = -1, second = -1;
    if (nn_d < DISTANCE_SQ_THRESHOLD) {
      closest = nn_idx;
      const int closest_ring = ring(corner_last[closest]);
      double best2 = DISTANCE_SQ_THRESHOLD;
      for (int j = closest + 1; j < n_corner_last; ++j) {  // increasing scan line (:312-335)
        if (ring(corner_last[j]) <= closest_ring) continue;
        if (ring(corner_last[j]) > (closest_ring + NEARBY_SCAN)) break;
        double d = sqdist_f(corner_last[j], sel);
        if (d < best2) { best2 = d; second = j; }
      }
      for (int j = closest - 1; j >= 0; --j) {  // decreasing scan line (:338-361)
        if (ring(corner_last[j]) >= closest_ring) continue;
        if (ring(corner_last[j]) < (closest_ring - NEARBY_SCAN)) break;
        double d = sqdist_f(corner_last[j], sel);
        if (d < best2) { best2 = d; second = j; }
      }
    }
    if (second >= 0) {  // :363-383 -- the residual takes the UNtransformed current point
      if (ccorr) ccorr->push_back({i, closest, second, -1});
      if (blocks) {
        const double cp[3] = {sharp[i].x, sharp[i].y, sharp[i].z};
        const double a[3] = {corner_last[closest].x, corner_last[closest].y, corner_last[closest].z};
        const double b[3] = {corner_last[second].x, corner_last[second].y, corner_last[second].z};
        blocks->push_back(make_edge(cp, a, b, ratio_of(sharp[i], distortion)));
      }
    }
  }

  for (int i = 0; i < (int)flat.size(); ++i) {  // :387
    PointXYZI sel = transform_to_start(flat[i], q, t, distortion);
    const float qq[3] = {sel.x, sel.y, sel.z};
    if (tree_surf.knn(qq, 1, &nn_idx, &nn_d) < 1) continue;
    if (!(nn_d < DISTANCE_SQ_THRESHOLD)) continue;
    const int closest = nn_idx;
    int m2 = -1, m3 = -1;
    const int closest_ring = ring(surf_last[closest]);
    double best2 = DISTANCE_SQ_THRESHOLD, best3 = DISTANCE_SQ_THRESHOLD;
    for (int j = closest + 1; j < n_surf_last; ++j) {  // :402-427
      if (ring(surf_last[j]) > (closest_ring + NEARBY_SCAN)) break;
      double d = sqdist_f(surf_last[j], sel);
      if (ring(surf_last[j]) <= closest_ring && d < best2) { best2 = d; m2 = j; }
      else if (ring(surf_last[j]) > closest_ring && d < best3) { best3 = d; m3 = j; }
    }
    for (int j = closest - 1; j >= 0; --j) {  // :430-455
      if (ring(surf_last[j]) < (closest_ring - NEARBY_SCAN)) break;
      double d = sqdist_f(surf_last[j], sel);
      if (ring(surf_last[j]) >= closest_ring && d < best2) { best2 = d; m2 = j; }
      else if (ring(surf_last[j]) < closest_ring && d < best3) { best3 = d; m3 = j; }
    }
    if (m2 >= 0 && m3 >= 0) {  // :457-481
      if (pcorr) pcorr->push_back({i, closest, m2, m3});
      if (blocks) {
        const double cp[3] = {flat[i].x, flat[i].y, flat[i].z};
        const double a[3] = {surf_last[closest].x, surf_last[closest].y, surf_last[closest].z};
        const double b[3] = {surf_last[m2].x, surf_last[m2].y, surf_last[m2].z};
        const double c[3] = {surf_last[m3].x, surf_last[m3].y, surf_last[m3].z};
        blocks->push_back(make_plane(cp, a, b, c, ratio_of(flat[i], distortion)));
      }
    }
  }
}

void Odometry::register_scan(const Cloud& sharp, const Cloud& flat, double q[4], double t[3], int outer_iters,
                             const SolveOptions& opt) {
  summaries.clear();
  times.assoc_ms = times.solve_ms = 0;
  for (int it = 0; it < outer_iters; ++it) {  // :278 opti_counter < 2
    std::vector<ResidualBlock> blocks;
    std::vector<Correspondence> cc, pc;
    double t0 = now_ms();
    associate(sharp, flat, q, t, &cc, &pc, &blocks);
    last_corner_corr = (int)cc.size(); last_plane_corr = (int)pc.size();
    times.assoc_ms += now_ms() - t0;
    t0 = now_ms();
    double x[7] = {q[0], q[1], q[2], q[3], t[0], t[1], t[2]};
    SolveSummary S;
    solve(blocks, x, opt, &S);
    for (int i = 0; i < 4; ++i) q[i] = x[i];
    for (int i = 0; i < 3; ++i) t[i] = x[4 + i];
    summaries.push_back(S);
    times.solve_ms += now_ms() - t0;
  }
}

void transform_to_end(const Cloud& in, const double qv[4], const double tv[3], bool distortion, Cloud* out) {
  const Quat q{qv[0], qv[1], qv[2], qv[3]};
  const Vec3 t{tv[0], tv[1], tv[2]};
  out->resize(in.size());
  for (size_t i = 0; i < in.size(); ++i) {
    const PointXYZI un = transform_to_start(in[i], q, t, distortion);          // :136-137 (rounded to float, as the PointType temp)
    const Vec3 d{(double)un.x - t.x, (double)un.y - t.y, (double)un.z - t.z};
    const Vec3 e = rotate(qinv(q), d);                                           // :140
    PointXYZI po;
    po.x = (float)e.x; po.y = (float)e.y; po.z = (float)e.z;
    po.intensity = (float)int(in[i].intensity);                                  // :147 remove distortion time info
    (*out)[i] = po;
  }
}

void integrate_pose(double q_w[4], double t_w[3], const double ql[4], const double tl[3]) {
  // :504-505  t_w_curr = t_w_curr + q_w_curr * t_last_curr ; q_w_curr = q_w_curr * q_last_curr
  Quat qw{q_w[0], q_w[1], q_w[2], q_w[3]}, q{ql[0], ql[1], ql[2], ql[3]};
  Vec3 r = rotate(qw, Vec3{tl[0], tl[1], tl[2]});
  t_w[0] += r.x; t_w[1] += r.y; t_w[2] += r.z;
  Quat o = qmul(qw, q);
  q_w[0] = o.x; q_w[1] = o.y; q_w[2] = o.z; q_w[3] = o.w;
}

}  // namespace orc
