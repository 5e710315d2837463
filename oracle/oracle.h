// ORACLE (test infrastructure, NOT product code).  PARITY: in-tree code pinned to the reference's own source text
// (oracle/_ref + tests/test_oracle_vs_reference_source.py), k-NN pinned to a real FLANN, Ceres / VoxelGrid / Eigen restated.  The reference
// (HKUST-Aerial-Robotics/A-LOAM @ e51f88c) ships no tests, golden vectors or fixtures, it cannot be
// compiled here (needs ROS + PCL + FLANN + Eigen + Ceres, none present, no network), and part of the
// arithmetic lives in un-vendored third-party code (Ceres 1.12.0, PCL 1.8.0 -- docker/Dockerfile:3-4;
// Eigen unpinned).  This directory is a dependency-free CPU restatement of the hot path, following the
// reference line by line where the code is in-tree and the libraries' published algorithms where not.
//
// What IS pinned: (1) every in-tree stage -- oracle/_ref compiles the reference's own lidarFactor.hpp, scanRegistration.cpp,
// laserOdometry.cpp and laserMapping.cpp unmodified against stand-in headers (oracle/ref_shim) and
// tests/test_oracle_vs_reference_source.py finds features.cc / odometry.cc / mapping.cc / cubemap.cc bit-identical to them;
// (2) the k-NN search (kdtree.cc) against a real FLANN build, the copy OpenCV vendors (tests/test_oracle_vs_flann.py).
// Ceres' minimiser, PCL's VoxelGrid and Eigen's decompositions remain restated from their published algorithms.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use it.
#pragma once
#include <cstdint>
#include <vector>
#include "smallmath.h"

namespace orc {

// pcl::PointXYZI carries 4 meaningful floats (x,y,z,intensity); PCL pads it to 32 B, we keep 16 B.
// include/aloam_velodyne/common.h:43
struct PointXYZI { float x, y, z, intensity; };
typedef std::vector<PointXYZI> Cloud;

// How the reference-internal UNSTABLE sorts are resolved (SURVEY.md 8a note 4):
//   LITERAL   : call std::sort with the reference's comparator (same libstdc++ introsort => the very
//               permutation the reference binary would produce on this input)
//   CANONICAL : order ties by original index ((key, index) lexicographic) -- the order the CUDA path defines
enum SortMode { SORT_LITERAL = 0, SORT_CANONICAL = 1 };

// ------------------------------------------------------------------ voxelgrid.cc  (pcl::VoxelGrid<PointXYZI>::applyFilter, PCL 1.8.0)
void voxel_grid(const Cloud& in, float leaf, SortMode mode, Cloud& out);

// ------------------------------------------------------------------ features.cc   (scanRegistration.cpp:85-112,129-408)
struct FeatureTimes { double prepare_ms, curvature_ms, sort_ms, pick_ms, voxel_ms, whole_ms; };
struct Features {
  Cloud full, sharp, less_sharp, flat, less_flat;
  std::vector<int> scan_start, scan_end;      // scanStartInd / scanEndInd
  std::vector<float> curvature;               // cloudCurvature[0..full.size())
  std::vector<int> label;                     // cloudLabel
  std::vector<int> picked;                    // cloudNeighborPicked (final state)
  FeatureTimes times;
};
// returns 0, or <0: -1 bad n_scans, -2 empty cloud after filtering, -3 too many points (>400000)
int extract_features(const float* xyz, int n, int stride_floats, int n_scans, double minimum_range,
                     SortMode mode, Features& out);

// ------------------------------------------------------------------ kdtree.cc     (pcl::KdTreeFLANN -> flann::KDTreeSingleIndex, leaf 15, L2_Simple<float>)
class KdTree {
 public:
  void build(const Cloud& cloud);
  // exact k-NN, ascending (dist, index); returns number found (min(k, size))
  int knn(const float q[3], int k, int* idx, float* sqdist) const;
  int size() const { return (int)pts_.size() / 3; }
 private:
  struct Node { int left, right; int divfeat; float divlow, divhigh; int child1, child2; };
  int divide(int left, int right, float bbox[6]);
  void search(int node, const float q[3], float mindistsq, float dists[3], int k, int& count,
              int* idx, float* sqd) const;
  std::vector<float> pts_;     // reordered x,y,z
  std::vector<int> vind_;      // reordered -> original index
  std::vector<Node> nodes_;
  float root_bbox_[6];
  int root_ = -1;
};

// ------------------------------------------------------------------ lm.cc         (lidarFactor.hpp:12-138 + ceres::Solve restatement, SURVEY.md 8a-R7)
enum FactorType { FACTOR_EDGE = 0, FACTOR_PLANE = 1, FACTOR_PLANE_NORM = 2 };
struct ResidualBlock {
  int type;
  double cp[3];   // curr_point
  double a[3];    // EDGE: last_point_a          PLANE: last_point_j    PLANE_NORM: plane_unit_norm
  double b[3];    // EDGE: last_point_b          PLANE: ljm_norm (precomputed in ctor, lidarFactor.hpp:64-65)
  double s;       // EDGE/PLANE: s               PLANE_NORM: negative_OA_dot_norm
  int rows() const { return type == FACTOR_EDGE ? 3 : 1; }
};
ResidualBlock make_edge(const double cp[3], const double a[3], const double b[3], double s);
ResidualBlock make_plane(const double cp[3], const double j[3], const double l[3], const double m[3], double s);
ResidualBlock make_plane_norm(const double cp[3], const double n[3], double d);

struct SolveOptions {   // the Ceres options the reference sets + the defaults it leaves (SURVEY.md R7)
  int max_num_iterations = 4;
  double huber_a = 0.1;
  double initial_trust_region_radius = 1e4, max_trust_region_radius = 1e16, min_trust_region_radius = 1e-32;
  double min_relative_decrease = 1e-3, min_lm_diagonal = 1e-6, max_lm_diagonal = 1e32;
  double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  int max_num_consecutive_invalid_steps = 5;
  bool jacobi_scaling = true;
  bool autodiff = true;       // true: Jet<7> through the literal functor text; false: closed-form Jacobian
};
struct IterationRecord { double cost, cost_change, gradient_max_norm, step_norm, relative_decrease, radius; int valid, successful; };
struct SolveSummary {
  double initial_cost = 0, final_cost = 0;
  int num_iterations = 0, num_successful_steps = 0, num_jacobian_evals = 0, num_cost_evals = 0;
  int termination = 0;   // 0 no_convergence(max iters) 1 gradient tol 2 parameter tol 3 function tol 4 empty problem 5 failure
  std::vector<IterationRecord> iters;
};
// Evaluate at x = [qx,qy,qz,qw,tx,ty,tz].  residuals (Huber-corrected), jacobian row-major rows x 6 in the
// tangent [dtheta(3), dt(3)], gradient (6) all optional.  Returns cost = sum 0.5*rho(|r_block|^2).
double evaluate(const std::vector<ResidualBlock>& blocks, const double x[7], double huber_a, bool autodiff,
                std::vector<double>* residuals, std::vector<double>* jacobian, double* gradient);
// JtJ (6x6 row-major), Jtr (6), cost at x -- what the CUDA K7 kernel produces.
double normal_equations(const std::vector<ResidualBlock>& blocks, const double x[7], double huber_a,
                        bool autodiff, double JtJ[36], double Jtr[6]);
void solve(const std::vector<ResidualBlock>& blocks, double x[7], const SolveOptions& opt, SolveSummary* summary);

// ------------------------------------------------------------------ odometry.cc   (laserOdometry.cpp:111-129,274-506,554-568)
struct Correspondence { int query; int a, b, c; };   // indices into the "last" clouds; c = -1 for edges
struct OdomTimes { double assoc_ms = 0, solve_ms = 0, tree_ms = 0; };
class Odometry {
 public:
  // laserOdometry.cpp:554-568 : swap in the less-sharp / less-flat clouds and rebuild the kd-trees
  void set_last(const Cloud& corner_last, const Cloud& surf_last);
  // laserOdometry.cpp:278-501 : outer_iters x (associate + ceres::Solve).  q = x,y,z,w (para_q), t (para_t), in/out.
  void register_scan(const Cloud& sharp, const Cloud& flat, double q[4], double t[3], int outer_iters,
                     const SolveOptions& opt);
  // one association pass at (q,t): laserOdometry.cpp:299-483
  void associate(const Cloud& sharp, const Cloud& flat, const double q[4], const double t[3],
                 std::vector<Correspondence>* corner_corr, std::vector<Correspondence>* plane_corr,
                 std::vector<ResidualBlock>* blocks) const;
  // #define DISTORTION (laserOdometry.cpp:59): 0 in the reference build; 1 = per-point interpolation ratio
  // s = (intensity - int(intensity)) / SCAN_PERIOD in TransformToStart (:115-116) and in the residual blocks (:376-379,470-473)
  bool distortion = false;
  // DISTANCE_SQ_THRESHOLD and NEARBY_SCAN (laserOdometry.cpp:65-66, constants there; aloam_config.dist_sq_thresh / nearby_scan)
  double dist_sq_thresh = 25, nearby_scan = 2.5;
  Cloud corner_last, surf_last;
  KdTree tree_corner, tree_surf;
  OdomTimes times;
  std::vector<SolveSummary> summaries;
  int last_corner_corr = 0, last_plane_corr = 0;
};
// laserOdometry.cpp:133-148 TransformToEnd (dead code in the reference: its only call sites sit under `if (0)`, :533-552)
void transform_to_end(const Cloud& in, const double q_last_curr[4], const double t_last_curr[3], bool distortion, Cloud* out);
// laserOdometry.cpp:504-505
void integrate_pose(double q_w[4], double t_w[3], const double q_last_curr[4], const double t_last_curr[3]);

// ------------------------------------------------------------------ mapping.cc    (laserMapping.cpp:142-173,542-734)
struct MapTimes { double tree_ms = 0, assoc_ms = 0, solve_ms = 0; };
struct MapFit { int query; int type; double p0[3]; double p1[3]; double d; int nn[5]; };  // edge: a,b ; plane: n,(unused),d
class Mapping {
 public:
  // laserMapping.cpp:531-539,558-559 : the gathered submap + kd-tree build
  void set_map(const Cloud& corner_map, const Cloud& surf_map);
  // laserMapping.cpp:554-729 : skip if map too thin; outer_iters x (5-NN + fit + ceres::Solve). x = parameters[7]
  // returns 1 if optimised, 0 if skipped (corner<=10 or surf<=50)
  int register_scan(const Cloud& corner_stack, const Cloud& surf_stack, double x[7], int outer_iters,
                    const SolveOptions& opt);
  void associate(const Cloud& corner_stack, const Cloud& surf_stack, const double x[7],
                 std::vector<MapFit>* fits, std::vector<ResidualBlock>* blocks) const;
  Cloud corner_map, surf_map;
  KdTree tree_corner, tree_surf;
  MapTimes times;
  std::vector<SolveSummary> summaries;
};
// laserMapping.cpp:142-152
void transform_associate_to_map(const double q_wmap_wodom[4], const double t_wmap_wodom[3],
                                const double q_wodom_curr[4], const double t_wodom_curr[3], double x[7]);
void transform_update(const double x[7], const double q_wodom_curr[4], const double t_wodom_curr[3],
                      double q_wmap_wodom[4], double t_wmap_wodom[3]);

// ------------------------------------------------------------------ cubemap.cc    (laserMapping.cpp:74-108,309-550,736-801)
// The 21 x 21 x 11 ring buffer of 50 m cubes and the whole per-frame mapping loop around it (SURVEY.md 8 f-1).
class CubeMap {
 public:
  CubeMap();
  // one frame of alaserMapping's process(): pose hand-off, shift, gather, stack filters, optimisation, insertion,
  // per-cube re-filter.  Returns 1 if the optimisation ran (map thick enough).  `pose` = parameters[7] afterwards.
  int step(const Cloud& corner_last, const Cloud& surf_last, const double q_wodom_curr[4], const double t_wodom_curr[3],
           float line_res, float plane_res, int outer_iters, const SolveOptions& opt, SortMode mode);
  std::vector<Cloud> corner, surf;        // laserCloudCornerArray / laserCloudSurfArray (4851 cubes each)
  int cen_w = 10, cen_h = 10, cen_d = 5;  // laserCloudCenWidth / Height / Depth
  double q_wmap_wodom[4] = {0, 0, 0, 1}, t_wmap_wodom[3] = {0, 0, 0};
  double pose[7] = {0, 0, 0, 1, 0, 0, 0};
  // state of the last step, for frame-by-frame parity checks
  std::vector<int> valid;                 // laserCloudValidInd
  Cloud corner_from_map, surf_from_map, corner_stack, surf_stack;
  int frames = 0;
 private:
  void shift_for(int& ci, int& cj, int& ck);
  void insert(const Cloud& stack, const double x[7], std::vector<Cloud>& cubes);
};

// 3x3 symmetric eigen (ascending eigenvalues, eigenvectors in columns, row-major V) -- Eigen::SelfAdjointEigenSolver stand-in
void eig3_sym(const double A[9], double evals[3], double V[9]);
// least squares solve of 5x3 A n = b by column-pivoted Householder QR (Eigen colPivHouseholderQr stand-in)
void lsq_5x3(const double A[15], const double b[5], double n[3]);

double now_ms();

}  // namespace orc
