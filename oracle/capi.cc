// ORACLE (test infrastructure) -- flat C interface over the oracle for ctypes (tests/, bench.py cpu_baseline leg,
// __graft_entry__.smoke()).  Not part of the product; the product C-ABI is include/aloam_b200.h.
#include <cstring>
#include "oracle.h"

using namespace orc;

namespace {
Cloud to_cloud(const float* p, int n) {
  Cloud c(n);
  if (n > 0) std::memcpy(c.data(), p, sizeof(PointXYZI) * (size_t)n);
  return c;
}
// packed residual block: 11 doubles  [type, cp(3), a(3), b(3), s]
const int kPack = 11;
void pack(const ResidualBlock& rb, double* o) {
  o[0] = rb.type;
  for (int i = 0; i < 3; ++i) { o[1 + i] = rb.cp[i]; o[4 + i] = rb.a[i]; o[7 + i] = rb.b[i]; }
  o[10] = rb.s;
}
ResidualBlock unpack(const double* o) {
  ResidualBlock rb; rb.type = (int)o[0];
  for (int i = 0; i < 3; ++i) { rb.cp[i] = o[1 + i]; rb.a[i] = o[4 + i]; rb.b[i] = o[7 + i]; }
  rb.s = o[10];
  return rb;
}
std::vector<ResidualBlock> unpack_all(const double* p, int n) {
  std::vector<ResidualBlock> v(n);
  for (int i = 0; i < n; ++i) v[i] = unpack(p + (size_t)i * kPack);
  return v;
}
SolveOptions make_opt(int max_iters, int autodiff, double huber) {
  SolveOptions o; o.max_num_iterations = max_iters; o.autodiff = autodiff != 0; o.huber_a = huber; return o;
}
// summary: [termination, num_iterations, num_successful, num_jac_evals, num_cost_evals, initial_cost, final_cost]
void put_summary(const SolveSummary& S, double* out) {
  if (!out) return;
  out[0] = S.termination; out[1] = S.num_iterations; out[2] = S.num_successful_steps;
  out[3] = S.num_jacobian_evals; out[4] = S.num_cost_evals; out[5] = S.initial_cost; out[6] = S.final_cost;
}
}  // namespace

extern "C" {

// ---------------------------------------------------------------- features
void* orc_features_extract(const float* xyz, int n, int stride, int n_scans, double min_range, int mode, int* err) {
  Features* f = new Features();
  int rc = extract_features(xyz, n, stride, n_scans, min_range, (SortMode)mode, *f);
  if (err) *err = rc;
  if (rc != 0) { delete f; return nullptr; }
  return f;
}
static const Cloud& pick_cloud(const Features* f, int which) {
  switch (which) { case 0: return f->full; case 1: return f->sharp; case 2: return f->less_sharp; case 3: return f->flat; default: return f->less_flat; }
}
int orc_features_size(void* h, int which) { return (int)pick_cloud((Features*)h, which).size(); }
void orc_features_copy(void* h, int which, float* out) {
  const Cloud& c = pick_cloud((Features*)h, which);
  if (!c.empty()) std::memcpy(out, c.data(), sizeof(PointXYZI) * c.size());
}
// which: 0 scan_start, 1 scan_end (n_scans ints) ; 2 label, 3 picked (full-size ints)
void orc_features_ints(void* h, int which, int* out) {
  Features* f = (Features*)h;
  const std::vector<int>& v = which == 0 ? f->scan_start : which == 1 ? f->scan_end : which == 2 ? f->label : f->picked;
  if (!v.empty()) std::memcpy(out, v.data(), sizeof(int) * v.size());
}
void orc_features_curvature(void* h, float* out) {
  Features* f = (Features*)h;
  if (!f->curvature.empty()) std::memcpy(out, f->curvature.data(), sizeof(float) * f->curvature.size());
}
void orc_features_times(void* h, double out[6]) {
  const FeatureTimes& t = ((Features*)h)->times;
  out[0] = t.prepare_ms; out[1] = t.curvature_ms; out[2] = t.sort_ms; out[3] = t.pick_ms; out[4] = t.voxel_ms; out[5] = t.whole_ms;
}
void orc_features_free(void* h) { delete (Features*)h; }

// ---------------------------------------------------------------- voxel grid (out capacity >= n points)
int orc_voxel_grid(const float* xyzi, int n, float leaf, int mode, float* out) {
  Cloud o;
  voxel_grid(to_cloud(xyzi, n), leaf, (SortMode)mode, o);
  if (!o.empty()) std::memcpy(out, o.data(), sizeof(PointXYZI) * o.size());
  return (int)o.size();
}

// ---------------------------------------------------------------- kd-tree
void* orc_kdtree_build(const float* xyzi, int n) { KdTree* t = new KdTree(); t->build(to_cloud(xyzi, n)); return t; }
void orc_kdtree_free(void* h) { delete (KdTree*)h; }
// queries: nq x qstride floats (x,y,z first) ; idx/sqd: nq x k ; missing entries = -1 / inf
void orc_kdtree_knn(void* h, const float* q, int nq, int qstride, int k, int* idx, float* sqd) {
  KdTree* t = (KdTree*)h;
  for (int i = 0; i < nq; ++i) {
    int c = t->knn(q + (size_t)i * qstride, k, idx + (size_t)i * k, sqd + (size_t)i * k);
    for (int j = c; j < k; ++j) { idx[(size_t)i * k + j] = -1; sqd[(size_t)i * k + j] = __builtin_inff(); }
  }
}
// brute force reference for the kd-tree itself (same float expression, (dist,index) order)
void orc_bruteforce_knn(const float* xyzi, int n, const float* q, int nq, int qstride, int k, int* idx, float* sqd) {
  for (int i = 0; i < nq; ++i) {
    const float* qq = q + (size_t)i * qstride;
    int* oi = idx + (size_t)i * k; float* od = sqd + (size_t)i * k;
    int count = 0;
    for (int p = 0; p < n; ++p) {
      float r = 0.f;
      float d0 = qq[0] - xyzi[4 * (size_t)p]; r += d0 * d0;
      float d1 = qq[1] - xyzi[4 * (size_t)p + 1]; r += d1 * d1;
      float d2 = qq[2] - xyzi[4 * (size_t)p + 2]; r += d2 * d2;
      if (count == k && !(r < od[k - 1])) continue;  // ascending p => equal distance never displaces
      int pos = count < k ? count : k - 1;
      if (count < k) ++count;
      while (pos > 0 && r < od[pos - 1]) { od[pos] = od[pos - 1]; oi[pos] = oi[pos - 1]; --pos; }
      od[pos] = r; oi[pos] = p;
    }
    for (int j = count; j < k; ++j) { oi[j] = -1; od[j] = __builtin_inff(); }
  }
}

// ---------------------------------------------------------------- residual blocks / LM
int orc_block_doubles() { return kPack; }
void orc_make_edge(const double cp[3], const double a[3], const double b[3], double s, double* out) { pack(make_edge(cp, a, b, s), out); }
void orc_make_plane(const double cp[3], const double j[3], const double l[3], const double m[3], double s, double* out) { pack(make_plane(cp, j, l, m, s), out); }
void orc_make_plane_norm(const double cp[3], const double n[3], double d, double* out) { pack(make_plane_norm(cp, n, d), out); }
double orc_normal_equations(const double* blocks, int n, const double x[7], double huber, int autodiff, double JtJ[36], double Jtr[6]) {
  return normal_equations(unpack_all(blocks, n), x, huber, autodiff != 0, JtJ, Jtr);
}
double orc_cost(const double* blocks, int n, const double x[7], double huber) {
  return evaluate(unpack_all(blocks, n), x, huber, true, nullptr, nullptr, nullptr);
}
// residuals (rows) and jacobian (rows x 6) ; returns rows
int orc_evaluate(const double* blocks, int n, const double x[7], double huber, int autodiff, double* residuals, double* jacobian, double* cost) {
  std::vector<double> r, J; double g[6];
  double c = evaluate(unpack_all(blocks, n), x, huber, autodiff != 0, &r, &J, g);
  if (cost) *cost = c;
  if (residuals) std::memcpy(residuals, r.data(), sizeof(double) * r.size());
  if (jacobian) std::memcpy(jacobian, J.data(), sizeof(double) * J.size());
  return (int)r.size();
}
// trace: up to max_trace rows of 8 doubles [cost, cost_change, gmax, step_norm, rel_decrease, radius, valid, successful]
int orc_solve(const double* blocks, int n, double x[7], int max_iters, int autodiff, double huber, double* summary7, double* trace, int max_trace) {
  SolveSummary S;
  solve(unpack_all(blocks, n), x, make_opt(max_iters, autodiff, huber), &S);
  put_summary(S, summary7);
  int rows = 0;
  if (trace)
    for (const IterationRecord& r : S.iters) {
      if (rows >= max_trace) break;
      double* o = trace + (size_t)rows * 8;
      o[0] = r.cost; o[1] = r.cost_change; o[2] = r.gradient_max_norm; o[3] = r.step_norm; o[4] = r.relative_decrease;
      o[5] = r.radius; o[6] = r.valid; o[7] = r.successful;
      ++rows;
    }
  return rows;
}
void orc_quat_plus(const double x[4], const double d[3], double out[4]) { quat_plus(x, d, out); }

// ---------------------------------------------------------------- odometry
void* orc_odom_create() { return new Odometry(); }
void orc_odom_free(void* h) { delete (Odometry*)h; }
void orc_odom_set_distortion(void* h, int on) { ((Odometry*)h)->distortion = on != 0; }
// DISTANCE_SQ_THRESHOLD and NEARBY_SCAN of the association (laserOdometry.cpp:65-66)
void orc_odom_set_params(void* h, double dist_sq_thresh, double nearby_scan) {
  Odometry* o = (Odometry*)h; o->dist_sq_thresh = dist_sq_thresh; o->nearby_scan = nearby_scan;
}
void orc_transform_to_end(const float* in, int n, const double q[4], const double t[3], int distortion, float* out) {
  Cloud o; transform_to_end(to_cloud(in, n), q, t, distortion != 0, &o);
  for (int i = 0; i < n; ++i) { out[4 * i] = o[i].x; out[4 * i + 1] = o[i].y; out[4 * i + 2] = o[i].z; out[4 * i + 3] = o[i].intensity; }
}
void orc_odom_set_last(void* h, const float* corner, int nc, const float* surf, int ns) {
  ((Odometry*)h)->set_last(to_cloud(corner, nc), to_cloud(surf, ns));
}
// corr_corner: n_sharp x 3 ints (query,a,b) ; corr_plane: n_flat x 4 ints (query,a,b,c) ; blocks: (n_sharp+n_flat) x 11 doubles
void orc_odom_associate(void* h, const float* sharp, int nsh, const float* flat, int nfl, const double q[4], const double t[3],
                        int* corr_corner, int* n_cc, int* corr_plane, int* n_pc, double* blocks, int* n_blocks) {
  std::vector<Correspondence> cc, pc; std::vector<ResidualBlock> bl;
  ((Odometry*)h)->associate(to_cloud(sharp, nsh), to_cloud(flat, nfl), q, t, &cc, &pc, &bl);
  if (corr_corner) for (size_t i = 0; i < cc.size(); ++i) { corr_corner[3 * i] = cc[i].query; corr_corner[3 * i + 1] = cc[i].a; corr_corner[3 * i + 2] = cc[i].b; }
  if (corr_plane) for (size_t i = 0; i < pc.size(); ++i) { corr_plane[4 * i] = pc[i].query; corr_plane[4 * i + 1] = pc[i].a; corr_plane[4 * i + 2] = pc[i].b; corr_plane[4 * i + 3] = pc[i].c; }
  if (blocks) for (size_t i = 0; i < bl.size(); ++i) pack(bl[i], blocks + i * kPack);
  if (n_cc) *n_cc = (int)cc.size();
  if (n_pc) *n_pc = (int)pc.size();
  if (n_blocks) *n_blocks = (int)bl.size();
}
// summaries: outer x 7 doubles ; times: [assoc_ms, solve_ms, tree_ms] ; counts: [corner_corr, plane_corr] of the last outer iter
void orc_odom_register(void* h, const float* sharp, int nsh, const float* flat, int nfl, double q[4], double t[3], int outer,
                       int max_iters, int autodiff, double huber, double* summaries, double times[3], int counts[2]) {
  Odometry* o = (Odometry*)h;
  o->register_scan(to_cloud(sharp, nsh), to_cloud(flat, nfl), q, t, outer, make_opt(max_iters, autodiff, huber));
  if (summaries) for (size_t i = 0; i < o->summaries.size(); ++i) put_summary(o->summaries[i], summaries + 7 * i);
  if (times) { times[0] = o->times.assoc_ms; times[1] = o->times.solve_ms; times[2] = o->times.tree_ms; }
  if (counts) { counts[0] = o->last_corner_corr; counts[1] = o->last_plane_corr; }
}
void orc_integrate_pose(double q_w[4], double t_w[3], const double q[4], const double t[3]) { integrate_pose(q_w, t_w, q, t); }

// ---------------------------------------------------------------- mapping
void* orc_map_create() { return new Mapping(); }
void orc_map_free(void* h) { delete (Mapping*)h; }
double orc_map_set_map(void* h, const float* corner, int nc, const float* surf, int ns) {
  Mapping* m = (Mapping*)h; m->set_map(to_cloud(corner, nc), to_cloud(surf, ns)); return m->times.tree_ms;
}
// fits: (nc+ns) rows of [query, type, p0(3), p1(3), d, nn(5)] = 14 doubles ; blocks packed
void orc_map_associate(void* h, const float* corner, int nc, const float* surf, int ns, const double x[7], double* fits, int* n_fits,
                       double* blocks, int* n_blocks) {
  std::vector<MapFit> f; std::vector<ResidualBlock> bl;
  ((Mapping*)h)->associate(to_cloud(corner, nc), to_cloud(surf, ns), x, &f, &bl);
  if (fits) for (size_t i = 0; i < f.size(); ++i) {
    double* o = fits + i * 14; o[0] = f[i].query; o[1] = f[i].type;
    for (int k = 0; k < 3; ++k) { o[2 + k] = f[i].p0[k]; o[5 + k] = f[i].p1[k]; }
    o[8] = f[i].d;
    for (int k = 0; k < 5; ++k) o[9 + k] = f[i].nn[k];
  }
  if (blocks) for (size_t i = 0; i < bl.size(); ++i) pack(bl[i], blocks + i * kPack);
  if (n_fits) *n_fits = (int)f.size();
  if (n_blocks) *n_blocks = (int)bl.size();
}
int orc_map_register(void* h, const float* corner, int nc, const float* surf, int ns, double x[7], int outer, int max_iters,
                     int autodiff, double huber, double* summaries, double times[3]) {
  Mapping* m = (Mapping*)h;
  int rc = m->register_scan(to_cloud(corner, nc), to_cloud(surf, ns), x, outer, make_opt(max_iters, autodiff, huber));
  if (summaries) for (size_t i = 0; i < m->summaries.size(); ++i) put_summary(m->summaries[i], summaries + 7 * i);
  if (times) { times[0] = m->times.assoc_ms; times[1] = m->times.solve_ms; times[2] = m->times.tree_ms; }
  return rc;
}
void orc_transform_associate_to_map(const double qm[4], const double tm[3], const double qo[4], const double to[3], double x[7]) {
  transform_associate_to_map(qm, tm, qo, to, x);
}
void orc_transform_update(const double x[7], const double qo[4], const double to[3], double qm[4], double tm[3]) {
  transform_update(x, qo, to, qm, tm);
}
void orc_eig3_sym(const double A[9], double ev[3], double V[9]) { eig3_sym(A, ev, V); }
void orc_lsq_5x3(const double A[15], const double b[5], double n[3]) { lsq_5x3(A, b, n); }

}  // extern "C"

// ------------------------------------------------------------------ cube store (cubemap.cc)
extern "C" {
void* orc_cubemap_create() { return new orc::CubeMap(); }
void orc_cubemap_free(void* h) { delete (orc::CubeMap*)h; }
// one mapping frame ; pose7 out ; info[0..5] = optimised, n valid cubes, corner_from_map, surf_from_map, corner_stack, surf_stack sizes
int orc_cubemap_step(void* h, const float* corner, int nc, const float* surf, int ns, const double q_odom[4], const double t_odom[3],
                     float line_res, float plane_res, int outer, int max_iters, double huber, int sort_mode, double pose7[7], int info[6]) {
  orc::CubeMap* m = (orc::CubeMap*)h;
  orc::SolveOptions opt; opt.max_num_iterations = max_iters; opt.huber_a = huber;
  orc::Cloud c(nc), s(ns);
  for (int i = 0; i < nc; ++i) c[i] = orc::PointXYZI{corner[4 * i], corner[4 * i + 1], corner[4 * i + 2], corner[4 * i + 3]};
  for (int i = 0; i < ns; ++i) s[i] = orc::PointXYZI{surf[4 * i], surf[4 * i + 1], surf[4 * i + 2], surf[4 * i + 3]};
  const int rc = m->step(c, s, q_odom, t_odom, line_res, plane_res, outer, opt, (orc::SortMode)sort_mode);
  for (int k = 0; k < 7; ++k) pose7[k] = m->pose[k];
  info[0] = rc; info[1] = (int)m->valid.size(); info[2] = (int)m->corner_from_map.size(); info[3] = (int)m->surf_from_map.size();
  info[4] = (int)m->corner_stack.size(); info[5] = (int)m->surf_stack.size();
  return rc;
}
// which: 0 corner_from_map, 1 surf_from_map, 2 corner_stack, 3 surf_stack ; returns the size, copies at most cap points
int orc_cubemap_get(void* h, int which, float* out, int cap) {
  orc::CubeMap* m = (orc::CubeMap*)h;
  const orc::Cloud& c = which == 0 ? m->corner_from_map : which == 1 ? m->surf_from_map : which == 2 ? m->corner_stack : m->surf_stack;
  const int n = (int)c.size();
  for (int i = 0; i < n && i < cap; ++i) { out[4 * i] = c[i].x; out[4 * i + 1] = c[i].y; out[4 * i + 2] = c[i].z; out[4 * i + 3] = c[i].intensity; }
  return n;
}
// cube bookkeeping: centre offsets, the valid cube indices of the last step, total stored points per type
void orc_cubemap_state(void* h, int cen[3], int* n_valid, int valid[125], long long totals[2], double q_wmap_wodom[4], double t_wmap_wodom[3]) {
  orc::CubeMap* m = (orc::CubeMap*)h;
  cen[0] = m->cen_w; cen[1] = m->cen_h; cen[2] = m->cen_d;
  *n_valid = (int)m->valid.size();
  for (size_t i = 0; i < m->valid.size() && i < 125; ++i) valid[i] = m->valid[i];
  totals[0] = totals[1] = 0;
  for (const auto& c : m->corner) totals[0] += (long long)c.size();
  for (const auto& c : m->surf) totals[1] += (long long)c.size();
  for (int k = 0; k < 4; ++k) q_wmap_wodom[k] = m->q_wmap_wodom[k];
  for (int k = 0; k < 3; ++k) t_wmap_wodom[k] = m->t_wmap_wodom[k];
}
// points of one cube (index i + 21 j + 441 k) ; which: 0 corner, 1 surf
int orc_cubemap_cube(void* h, int which, int index, float* out, int cap) {
  orc::CubeMap* m = (orc::CubeMap*)h;
  if (index < 0 || index >= 21 * 21 * 11) return -1;
  const orc::Cloud& c = which == 0 ? m->corner[index] : m->surf[index];
  const int n = (int)c.size();
  for (int i = 0; i < n && i < cap; ++i) { out[4 * i] = c[i].x; out[4 * i + 1] = c[i].y; out[4 * i + 2] = c[i].z; out[4 * i + 3] = c[i].intensity; }
  return n;
}
}
