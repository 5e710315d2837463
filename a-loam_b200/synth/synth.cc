// Synthetic lidar world + sensor models (deterministic, seeded).
//
// Not a restatement of anything in the reference: A-LOAM ships no data and no generator
// (kittiHelper.cpp only replays KITTI files).  This is the "synthetic data of that shape" the
// benchmark contract asks for.  The sensor models are derived from the reference's own ring
// formulas so that every generated beam lands on the ring the reference would assign it:
//   VLP-16  scanRegistration.cpp:171   id = int((angle + 15) / 2 + 0.5)
//   HDL-32  scanRegistration.cpp:180   id = int((angle + 92/3) * 3/4)            (truncating!)
//   HDL-64  scanRegistration.cpp:189-199  two blocks, keep id 0..50, -24.33 <= angle <= 2
// Points are emitted in firing order (azimuth-major, clockwise so that -atan2(y,x) increases,
// scanRegistration.cpp:141-153,208), no-return rays are dropped, range noise is Gaussian along
// the ray (so the elevation angle -- hence the ring -- is unaffected by the noise).  synth_scan_beams replaces the nominal
// beams with a table of its own (calibration offsets, lasers off the sensor origin) whose returns do land on and across
// the ring edges.
//
// World: an "urban canyon" made only of a ground plane and axis-aligned boxes, so every ray is
// intersected in closed form.
//
// C interface (ctypes-friendly), see bottom of file.

#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>
#include <algorithm>

namespace {

struct Rng {  // splitmix64 -> uniform / gaussian; platform independent except libm log/cos
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
  double uniform(double a, double b) { return a + (b - a) * uniform(); }
  double gauss() {
    double u1 = uniform(), u2 = uniform();
    if (u1 < 1e-300) u1 = 1e-300;
    return std::sqrt(-2.0 * std::log(u1)) * std::cos(6.283185307179586 * u2);
  }
};

struct Box { double lo[3], hi[3]; };

struct World {
  std::vector<Box> boxes;
  double ground_z;
};

void add_box(World& w, double x0, double x1, double y0, double y1, double z0, double z1) {
  Box b; b.lo[0] = x0; b.hi[0] = x1; b.lo[1] = y0; b.hi[1] = y1; b.lo[2] = z0; b.hi[2] = z1;
  w.boxes.push_back(b);
}

World make_world(uint64_t seed) {
  World w; w.ground_z = -1.8;
  const double gz = w.ground_z;
  // long walls y = +-12, split every 20 m with a 2 m gap (vertical edges at the gap jambs)
  for (int k = -16; k < 16; ++k) {
    double x0 = 20.0 * k + 1.0, x1 = 20.0 * k + 19.0;
    add_box(w, x0, x1, 12.0, 12.5, gz, gz + 6.0);
    add_box(w, x0, x1, -12.5, -12.0, gz, gz + 6.0);
  }
  // a second, taller facade behind the gaps so rays through the gaps still return
  add_box(w, -330.0, 330.0, 18.0, 18.5, gz, gz + 9.0);
  add_box(w, -330.0, 330.0, -18.5, -18.0, gz, gz + 9.0);
  // cross walls every 40 m with a 6 m door gap in the middle
  for (int k = -8; k < 8; ++k) {
    double x = 40.0 * k + 20.0;
    add_box(w, x, x + 0.5, 3.0, 12.0, gz, gz + 6.0);
    add_box(w, x, x + 0.5, -12.0, -3.0, gz, gz + 6.0);
  }
  // 0.4 m square poles, 5 m tall, on a 10 m lattice either side of the path
  for (int k = -30; k < 30; ++k) {
    double x = 10.0 * k + 5.0;
    add_box(w, x - 0.2, x + 0.2, 6.8, 7.2, gz, gz + 5.0);
    add_box(w, x - 0.2, x + 0.2, -7.2, -6.8, gz, gz + 5.0);
  }
  // box clutter (seeded)
  Rng rng(seed * 7919u + 17u);
  for (int i = 0; i < 160; ++i) {
    double cx = rng.uniform(-300.0, 300.0);
    double side = rng.uniform() < 0.5 ? 1.0 : -1.0;
    double cy = side * rng.uniform(3.0, 10.5);
    double sx = rng.uniform(0.5, 2.5), sy = rng.uniform(0.5, 2.0), sz = rng.uniform(0.5, 2.5);
    add_box(w, cx - sx / 2, cx + sx / 2, cy - sy / 2, cy + sy / 2, gz, gz + sz);
  }
  return w;
}

// nearest hit of ray o + t d, t in (tmin, tmax); returns tmax if none
inline double cast(const World& w, const std::vector<int>& cand, const double o[3], const double d[3],
                   double tmin, double tmax) {
  double best = tmax;
  if (d[2] < -1e-12) {
    double t = (w.ground_z - o[2]) / d[2];
    if (t > tmin && t < best) best = t;
  }
  double inv[3];
  for (int a = 0; a < 3; ++a) inv[a] = 1.0 / (std::fabs(d[a]) < 1e-300 ? (d[a] < 0 ? -1e-300 : 1e-300) : d[a]);
  for (int bi : cand) {
    const Box& b = w.boxes[bi];
    double t0 = tmin, t1 = best;
    bool hit = true;
    for (int a = 0; a < 3; ++a) {
      double ta = (b.lo[a] - o[a]) * inv[a], tb = (b.hi[a] - o[a]) * inv[a];
      if (ta > tb) std::swap(ta, tb);
      if (ta > t0) t0 = ta;
      if (tb < t1) t1 = tb;
      if (t0 > t1) { hit = false; break; }
    }
    if (hit && t0 > tmin && t0 < best) best = t0;
  }
  return best;
}

struct Pose { double R[9]; double t[3]; double q[4]; };  // R row-major, q = x,y,z,w

void quat_from_rpy(double roll, double pitch, double yaw, double q[4]) {
  double cr = std::cos(roll / 2), sr = std::sin(roll / 2);
  double cp = std::cos(pitch / 2), sp = std::sin(pitch / 2);
  double cy = std::cos(yaw / 2), sy = std::sin(yaw / 2);
  q[3] = cr * cp * cy + sr * sp * sy;
  q[0] = sr * cp * cy - cr * sp * sy;
  q[1] = cr * sp * cy + sr * cp * sy;
  q[2] = cr * cp * sy - sr * sp * cy;
}

void rot_from_quat(const double q[4], double R[9]) {
  double x = q[0], y = q[1], z = q[2], w = q[3];
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}

// Trajectory: 0.8 m / scan along heading, yaw +1 deg / scan, small roll/pitch sinusoid.
Pose trajectory_pose(int k) {
  Pose P;
  double x = 0, y = 0, yaw = 0;
  for (int i = 0; i < k; ++i) {
    x += 0.8 * std::cos(yaw); y += 0.8 * std::sin(yaw);
    yaw += 0.25 * M_PI / 180.0 * (((i / 8) % 2) ? -1.0 : 1.0) * 4.0;  // +-1 deg/scan, sign flips every 8 scans
  }
  double roll = 0.004 * std::sin(0.7 * k), pitch = 0.003 * std::sin(0.45 * k + 0.3);
  quat_from_rpy(roll, pitch, yaw, P.q);
  rot_from_quat(P.q, P.R);
  P.t[0] = x; P.t[1] = y; P.t[2] = 0.0;
  return P;
}

int sensor_elevations(int n_scans, std::vector<double>& elev_deg) {
  elev_deg.clear();
  if (n_scans == 16) {
    for (int k = 0; k < 16; ++k) elev_deg.push_back(-15.0 + 2.0 * k);
  } else if (n_scans == 32) {
    for (int k = 0; k < 32; ++k) elev_deg.push_back(-92.0 / 3.0 + (k + 0.5) * 4.0 / 3.0);
  } else if (n_scans == 64) {
    // whole pattern shifted by -0.04 deg so ring 0 is not sliced by the "angle > 2" cut
    for (int k = 0; k < 32; ++k) elev_deg.push_back(1.96 - k / 3.0);
    for (int m = 0; m < 32; ++m) elev_deg.push_back(-8.87 - 0.5 * m);
  } else {
    return -1;
  }
  return 0;
}

// Where a sweep is cut and how it is fired.  The neutral value is the layout of synth_scan.
//   start_col  azimuth of the first firing column, in columns: phi = pi - 2 pi (start_col +- j + 0.37) / n_az
//   n_col      number of firing columns (n_az = one revolution)
//   ring_off   per-beam azimuth offset [deg] added to the firing azimuth (nullptr = none); the world is not moved
//   laser_major  emit beam by beam (all columns of beam 0, then beam 1, ...) instead of column by column
//   ccw        the firing azimuth rises with j (-atan2(y, x) falls) instead of falling
//   n_beams, elev, z_off  a beam table instead of the sensor's nominal one (elev == nullptr): n_beams lasers (any count, not
//              tied to n_scans) at elevations elev[b] [deg], each firing from (0, 0, z_off[b]) [m] in the sensor frame
//              (z_off may be null).  A laser origin off the sensor origin makes the elevation seen from the origin -- the one
//              the reference bins -- change with range, so one laser's returns can fall on either side of a ring edge.
struct Layout {
  double start_col = 0.0;
  int n_col = 0;
  const double* ring_off = nullptr;
  int laser_major = 0, ccw = 0;
  int n_beams = 0;
  const double* elev = nullptr;
  const double* z_off = nullptr;
};

// ring id of a return as scanRegistration.cpp:166-205 assigns it, or -1 when it drops the return
int reference_ring(float x, float y, float z, int n_scans) {
  const float angle = (float)(std::atan((double)z / std::sqrt((double)(x * x + y * y))) * 180 / M_PI);
  int id;
  if (n_scans == 16) {
    id = int((angle + 15) / 2 + 0.5);
    return (id > n_scans - 1 || id < 0) ? -1 : id;
  }
  if (n_scans == 32) {
    id = int((angle + 92.0 / 3.0) * 3.0 / 4.0);
    return (id > n_scans - 1 || id < 0) ? -1 : id;
  }
  if (angle >= -8.83) id = int((2 - angle) * 3.0 + 0.5);
  else id = n_scans / 2 + int((-8.83 - angle) * 2.0 + 0.5);
  return (angle > 2 || angle < -24.33 || id > 50 || id < 0) ? -1 : id;
}

// The azimuth fix-ups of scanRegistration.cpp:141-153 and :208-236 compare float -atan2f(y, x) with thresholds.  Host and
// device atan2f differ in the last ulp, so a return closer than kSeamMargin to a threshold it is tested against could take
// the other branch on the GPU.  Replays the reference's walk over the surviving returns and returns -3 if one is that close
// (a return near the half-sweep test is checked against the thresholds of both halves, since the flag may flip there).
// n_scans = 0: every surviving return takes part in the walk (rings from the driver, not from a formula).
constexpr double kSeamMargin = 1e-5;
int check_seam_margins(const float* pts, int n, int n_scans, double minimum_range) {
  const float thres = (float)minimum_range;
  std::vector<int> keep;
  for (int i = 0; i < n; ++i) {
    const float* p = pts + (size_t)i * 4;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] < thres * thres) continue;
    keep.push_back(i);
  }
  if (keep.empty()) return 0;
  auto ori_of = [&](int i) { return -std::atan2(pts[(size_t)i * 4 + 1], pts[(size_t)i * 4]); };
  const float start = ori_of(keep.front());
  const float end_raw = ori_of(keep.back()) + 2 * M_PI;
  auto near = [](double a, double b) { return std::fabs(a - b) < kSeamMargin; };
  if (near(end_raw - start, 3 * M_PI) || near(end_raw - start, M_PI)) return -3;
  float end = end_raw;
  if (end - start > 3 * M_PI) end -= 2 * M_PI;
  else if (end - start < M_PI) end += 2 * M_PI;
  bool half = false;
  for (int i : keep) {
    const float* p = pts + (size_t)i * 4;
    if (n_scans > 0 && reference_ring(p[0], p[1], p[2], n_scans) < 0) continue;   // dropped before the azimuth walk (:174-175)
    float ori = ori_of(i);
    const bool pre_near = near(ori, start - M_PI / 2) || near(ori, start + M_PI * 3 / 2);
    const bool post_near = near(ori + 2 * M_PI, end - M_PI * 3 / 2) || near(ori + 2 * M_PI, end + M_PI / 2);
    if (!half) {
      if (ori < start - M_PI / 2) ori += 2 * M_PI;
      else if (ori > start + M_PI * 3 / 2) ori -= 2 * M_PI;
      const bool at_half = near(ori - start, M_PI);
      if (pre_near || (at_half && post_near)) return -3;
      if (ori - start > M_PI) half = true;
    } else if (post_near) {
      return -3;
    }
  }
  return 0;
}

// beam_out (may be null): the beam index of every return written
int generate(uint64_t seed, int n_scans, int n_az, int scan_index, double noise_sigma, double max_range, const Layout& lay,
             float* out, int* beam_out, int capacity) {
  std::vector<double> elev;
  if (lay.elev) {
    if (lay.n_beams <= 0) return -2;
    elev.assign(lay.elev, lay.elev + lay.n_beams);
  } else if (sensor_elevations(n_scans, elev) != 0) {
    return -1;
  }
  const int nb = (int)elev.size();
  const int n_col = lay.n_col;
  if (n_az <= 0 || n_col <= 0 || capacity < nb * n_col) return -2;
  World w = make_world(seed);
  Pose P = trajectory_pose(scan_index);
  // candidate boxes within range
  std::vector<int> cand;
  for (size_t i = 0; i < w.boxes.size(); ++i) {
    const Box& b = w.boxes[i];
    double dx = std::max({b.lo[0] - P.t[0], 0.0, P.t[0] - b.hi[0]});
    double dy = std::max({b.lo[1] - P.t[1], 0.0, P.t[1] - b.hi[1]});
    if (dx * dx + dy * dy < (max_range + 1) * (max_range + 1)) cand.push_back((int)i);
  }
  std::vector<float> tmp((size_t)nb * n_col * 4);
  std::vector<uint8_t> ok((size_t)nb * n_col, 0);
  unsigned nthreads = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
  auto work = [&](int j0, int j1) {
    for (int j = j0; j < j1; ++j) {
      // per-column rng so the result does not depend on the thread count
      Rng rng(seed * 1000003ull + (uint64_t)scan_index * 7907ull + (uint64_t)j * 104729ull + 12345ull);
      const double col = lay.ccw ? lay.start_col - j : j + lay.start_col;
      double phi = M_PI - 2.0 * M_PI * (col + 0.37) / n_az;  // clockwise unless ccw
      double cph = std::cos(phi), sph = std::sin(phi);
      for (int b = 0; b < nb; ++b) {
        if (lay.ring_off) {
          const double pb = phi + lay.ring_off[b] * M_PI / 180.0;
          cph = std::cos(pb); sph = std::sin(pb);
        }
        double el = elev[b] * M_PI / 180.0;
        double ds[3] = {std::cos(el) * cph, std::cos(el) * sph, std::sin(el)};
        double d[3] = {P.R[0] * ds[0] + P.R[1] * ds[1] + P.R[2] * ds[2],
                       P.R[3] * ds[0] + P.R[4] * ds[1] + P.R[5] * ds[2],
                       P.R[6] * ds[0] + P.R[7] * ds[1] + P.R[8] * ds[2]};
        double t, r;
        size_t o = lay.laser_major ? (size_t)b * n_col + j : (size_t)j * nb + b;
        if (lay.elev) {  // the laser fires from (0, 0, dz) of the sensor frame
          const double dz = lay.z_off ? lay.z_off[b] : 0.0;
          const double org[3] = {P.t[0] + P.R[2] * dz, P.t[1] + P.R[5] * dz, P.t[2] + P.R[8] * dz};
          t = cast(w, cand, org, d, 0.05, max_range);
          const double nz = rng.gauss();
          if (t >= max_range) continue;
          r = t + noise_sigma * nz;
          tmp[o * 4 + 2] = (float)(dz + r * ds[2]);
        } else {
          t = cast(w, cand, P.t, d, 0.05, max_range);
          const double nz = rng.gauss();  // always drawn, so streams stay aligned
          if (t >= max_range) continue;
          r = t + noise_sigma * nz;
          tmp[o * 4 + 2] = (float)(r * ds[2]);
        }
        tmp[o * 4 + 0] = (float)(r * ds[0]);
        tmp[o * 4 + 1] = (float)(r * ds[1]);
        tmp[o * 4 + 3] = 0.0f;
        ok[o] = 1;
      }
    }
  };
  std::vector<std::thread> th;
  int per = (n_col + (int)nthreads - 1) / (int)nthreads;
  for (unsigned i = 0; i < nthreads; ++i) {
    int j0 = (int)i * per, j1 = std::min(n_col, j0 + per);
    if (j0 < j1) th.emplace_back(work, j0, j1);
  }
  for (auto& t : th) t.join();
  int n = 0;
  for (size_t o = 0; o < ok.size(); ++o)
    if (ok[o]) {
      std::memcpy(out + (size_t)n * 4, &tmp[o * 4], 16);
      if (beam_out) beam_out[n] = lay.laser_major ? (int)(o / n_col) : (int)(o % nb);
      ++n;
    }
  return n;
}

}  // namespace

extern "C" {

// Ground-truth pose of scan k in the world: q = x,y,z,w ; t.
void synth_pose(int k, double q[4], double t[3]) {
  Pose P = trajectory_pose(k);
  for (int i = 0; i < 4; ++i) q[i] = P.q[i];
  for (int i = 0; i < 3; ++i) t[i] = P.t[i];
}

// Generate scan `scan_index` of sensor `n_scans` (16/32/64) with `n_az` azimuth steps.
// out: up to n_scans*n_az points, 4 floats each (x,y,z,0) in the SENSOR frame, firing order.
// Returns the number of points written, or <0 on error.
int synth_scan(uint64_t seed, int n_scans, int n_az, int scan_index, double noise_sigma,
               double max_range, float* out, int capacity) {
  Layout lay;
  lay.n_col = n_az;
  return generate(seed, n_scans, n_az, scan_index, noise_sigma, max_range, lay, out, nullptr, capacity);
}

// The same scan cut and fired differently (see Layout): n_col columns from start_col, per-beam azimuth offsets ring_off_deg
// (n_scans entries, may be null), beam-major order, counter-clockwise rotation.  Returns -3 when a surviving return lies
// within kSeamMargin of an azimuth threshold of the reference's sweep walk (minimum_range decides what survives).
int synth_scan_seam(uint64_t seed, int n_scans, int n_az, int scan_index, double noise_sigma, double max_range,
                    double start_col, int n_col, const double* ring_off_deg, int laser_major, int ccw, double minimum_range,
                    float* out, int capacity) {
  Layout lay;
  lay.start_col = start_col; lay.n_col = n_col; lay.ring_off = ring_off_deg; lay.laser_major = laser_major; lay.ccw = ccw;
  const int n = generate(seed, n_scans, n_az, scan_index, noise_sigma, max_range, lay, out, nullptr, capacity);
  if (n < 0) return n;
  const int rc = check_seam_margins(out, n, n_scans, minimum_range);
  return rc ? rc : n;
}

// synth_scan_seam with a beam table of its own (see Layout): n_beams lasers at elev_deg[b] firing from (0, 0, z_off_m[b])
// (z_off_m may be null), per-beam azimuth offsets ring_off_deg (n_beams entries, may be null).  The rings are still binned
// by the reference's n_scans formula.  beam_out (may be null) receives the laser of every return.  Returns -3 like
// synth_scan_seam.  Capacity: n_beams * n_col returns.
int synth_scan_beams(uint64_t seed, int n_scans, int n_az, int scan_index, double noise_sigma, double max_range,
                     double start_col, int n_col, int n_beams, const double* elev_deg, const double* z_off_m,
                     const double* ring_off_deg, int laser_major, int ccw, double minimum_range, float* out, int* beam_out,
                     int capacity) {
  if (!elev_deg) return -2;
  Layout lay;
  lay.start_col = start_col; lay.n_col = n_col; lay.ring_off = ring_off_deg; lay.laser_major = laser_major; lay.ccw = ccw;
  lay.n_beams = n_beams; lay.elev = elev_deg; lay.z_off = z_off_m;
  const int n = generate(seed, n_scans, n_az, scan_index, noise_sigma, max_range, lay, out, beam_out, capacity);
  if (n < 0) return n;
  const int rc = check_seam_margins(out, n, n_scans, minimum_range);
  return rc ? rc : n;
}

// A sensor that reports each return's ring (a driver's `ring` field): n_beams lasers at elev_deg[b], laser b's returns carry
// ring_of_beam[b] in float 3.  Cut and fired like synth_scan_seam (ring_off_deg: n_beams entries, may be null).  No formula
// drops a return, so the seam margins are checked on every return that survives minimum_range (-3 like synth_scan_seam).
int synth_scan_rings(uint64_t seed, int n_az, int scan_index, double noise_sigma, double max_range, double start_col, int n_col,
                     int n_beams, const double* elev_deg, const int* ring_of_beam, const double* ring_off_deg, int laser_major, int ccw,
                     double minimum_range, float* out, int capacity) {
  if (!elev_deg || !ring_of_beam || n_beams <= 0) return -2;
  Layout lay;
  lay.start_col = start_col; lay.n_col = n_col; lay.ring_off = ring_off_deg; lay.laser_major = laser_major; lay.ccw = ccw;
  lay.n_beams = n_beams; lay.elev = elev_deg;
  std::vector<int> beam((size_t)std::max(capacity, 0));
  const int n = generate(seed, 0, n_az, scan_index, noise_sigma, max_range, lay, out, beam.data(), capacity);
  if (n < 0) return n;
  for (int i = 0; i < n; ++i) out[(size_t)i * 4 + 3] = (float)ring_of_beam[beam[i]];
  const int rc = check_seam_margins(out, n, 0, minimum_range);
  return rc ? rc : n;
}

}  // extern "C"
