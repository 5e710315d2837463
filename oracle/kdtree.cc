// ORACLE (test infrastructure) -- exact k-NN the way pcl::KdTreeFLANN<PointXYZI> provides it to
// laserOdometry.cpp:302,390,567-568 and laserMapping.cpp:558-559,582,648: the cloud's x,y,z are copied to a
// float array and indexed by flann::KDTreeSingleIndex (leaf_max_size 15, reorder = true, L2_Simple<float>);
// nearestKSearch is exact (eps = 0), results ascending, distance = ((dx*dx) + dy*dy) + dz*dz in float.
// FLANN/PCL are not in /root/reference (un-vendored); this follows FLANN's published kdtree_single_index.h
// (middle-split on the widest bbox dimension, branch-and-bound on per-dimension box distances).
// Deviation, declared: FLANN resolves exact-distance ties by traversal order; here ties are resolved by the
// smaller original index so that the result is a function of the input only (SURVEY.md 8a "KD").
// PINNED (the one part of the oracle that is): tests/test_oracle_vs_flann.py compares this file with a real FLANN
// build -- the copy OpenCV vendors, cv2.flann_Index with KDTREE_SINGLE / leaf_max_size 15 -- on random clouds and on
// the searches of both registration stages: identical neighbour lists (tie rows as sets), bit-identical distances.
#include <algorithm>
#include <cmath>
#include "oracle.h"

namespace orc {

namespace {
const int kLeafMax = 15;

inline bool better(float d, int i, float d2, int i2) { return d < d2 || (d == d2 && i < i2); }
}  // namespace

void KdTree::build(const Cloud& cloud) {
  const int n = (int)cloud.size();
  nodes_.clear();
  vind_.resize(n);
  std::vector<float> raw((size_t)n * 3);
  for (int i = 0; i < n; ++i) {
    vind_[i] = i;
    raw[3 * (size_t)i] = cloud[i].x; raw[3 * (size_t)i + 1] = cloud[i].y; raw[3 * (size_t)i + 2] = cloud[i].z;
  }
  pts_.swap(raw);  // temporarily un-reordered; divide() permutes vind_ only
  root_ = -1;
  if (n == 0) { pts_.clear(); return; }
  for (int a = 0; a < 3; ++a) { root_bbox_[2 * a] = pts_[a]; root_bbox_[2 * a + 1] = pts_[a]; }
  for (int i = 1; i < n; ++i)
    for (int a = 0; a < 3; ++a) {
      float v = pts_[3 * (size_t)i + a];
      if (v < root_bbox_[2 * a]) root_bbox_[2 * a] = v;
      if (v > root_bbox_[2 * a + 1]) root_bbox_[2 * a + 1] = v;
    }
  float bbox[6];
  for (int i = 0; i < 6; ++i) bbox[i] = root_bbox_[i];
  nodes_.reserve((size_t)n / 4 + 16);
  root_ = divide(0, n, bbox);
  // reorder = true: gather points in leaf order for locality
  std::vector<float> re((size_t)n * 3);
  for (int i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) re[3 * (size_t)i + a] = pts_[3 * (size_t)vind_[i] + a];
  pts_.swap(re);
}

int KdTree::divide(int left, int right, float bbox[6]) {
  const int me = (int)nodes_.size();
  nodes_.push_back(Node());
  auto coord = [&](int k, int a) { return pts_[3 * (size_t)vind_[k] + a]; };
  if (right - left <= kLeafMax) {
    nodes_[me].child1 = nodes_[me].child2 = -1;
    nodes_[me].left = left; nodes_[me].right = right;
    for (int a = 0; a < 3; ++a) { bbox[2 * a] = coord(left, a); bbox[2 * a + 1] = coord(left, a); }
    for (int k = left + 1; k < right; ++k)
      for (int a = 0; a < 3; ++a) {
        float v = coord(k, a);
        if (v < bbox[2 * a]) bbox[2 * a] = v;
        if (v > bbox[2 * a + 1]) bbox[2 * a + 1] = v;
      }
    return me;
  }
  // middleSplit_: widest bbox dimension (among near-ties the one with the widest data spread)
  const float EPS = 0.00001f;
  float max_span = bbox[1] - bbox[0];
  for (int a = 1; a < 3; ++a) max_span = std::max(max_span, bbox[2 * a + 1] - bbox[2 * a]);
  float max_spread = -1.f;
  int cutfeat = 0;
  auto minmax = [&](int a, float& mn, float& mx) {
    mn = mx = coord(left, a);
    for (int k = left + 1; k < right; ++k) { float v = coord(k, a); if (v < mn) mn = v; if (v > mx) mx = v; }
  };
  for (int a = 0; a < 3; ++a) {
    float span = bbox[2 * a + 1] - bbox[2 * a];
    if (span > (1 - EPS) * max_span) {
      float mn, mx; minmax(a, mn, mx);
      if (mx - mn > max_spread) { cutfeat = a; max_spread = mx - mn; }
    }
  }
  float split_val = (bbox[2 * cutfeat] + bbox[2 * cutfeat + 1]) / 2;
  float mn, mx; minmax(cutfeat, mn, mx);
  float cutval = split_val < mn ? mn : (split_val > mx ? mx : split_val);
  // planeSplit: [left,lim1) < cutval ; [lim1,lim2) == cutval ; [lim2,right) > cutval
  int count = right - left;
  int* ind = vind_.data() + left;
  int l = 0, r = count - 1;
  for (;;) {
    while (l <= r && pts_[3 * (size_t)ind[l] + cutfeat] < cutval) ++l;
    while (l <= r && pts_[3 * (size_t)ind[r] + cutfeat] >= cutval) --r;
    if (l > r) break;
    std::swap(ind[l], ind[r]); ++l; --r;
  }
  int lim1 = l;
  r = count - 1;
  for (;;) {
    while (l <= r && pts_[3 * (size_t)ind[l] + cutfeat] <= cutval) ++l;
    while (l <= r && pts_[3 * (size_t)ind[r] + cutfeat] > cutval) --r;
    if (l > r) break;
    std::swap(ind[l], ind[r]); ++l; --r;
  }
  int lim2 = l;
  int idx;
  if (lim1 > count / 2) idx = lim1;
  else if (lim2 < count / 2) idx = lim2;
  else idx = count / 2;

  float lb[6], rb[6];
  for (int i = 0; i < 6; ++i) { lb[i] = bbox[i]; rb[i] = bbox[i]; }
  lb[2 * cutfeat + 1] = cutval;
  rb[2 * cutfeat] = cutval;
  int c1 = divide(left, left + idx, lb);
  int c2 = divide(left + idx, right, rb);
  nodes_[me].divfeat = cutfeat;
  nodes_[me].divlow = lb[2 * cutfeat + 1];
  nodes_[me].divhigh = rb[2 * cutfeat];
  nodes_[me].child1 = c1; nodes_[me].child2 = c2;
  nodes_[me].left = left; nodes_[me].right = right;
  for (int a = 0; a < 3; ++a) {
    bbox[2 * a] = std::min(lb[2 * a], rb[2 * a]);
    bbox[2 * a + 1] = std::max(lb[2 * a + 1], rb[2 * a + 1]);
  }
  return me;
}

void KdTree::search(int ni, const float q[3], float mindistsq, float dists[3], int k, int& count, int* idx,
                    float* sqd) const {
  const Node& nd = nodes_[ni];
  if (nd.child1 < 0) {
    for (int i = nd.left; i < nd.right; ++i) {
      const float* p = &pts_[3 * (size_t)i];
      float result = 0.f;  // L2_Simple: result += diff*diff, x then y then z
      float d0 = q[0] - p[0]; result += d0 * d0;
      float d1 = q[1] - p[1]; result += d1 * d1;
      float d2 = q[2] - p[2]; result += d2 * d2;
      const int oi = vind_[i];
      if (count == k && !better(result, oi, sqd[k - 1], idx[k - 1])) continue;
      int pos = count < k ? count : k - 1;
      if (count < k) ++count;
      while (pos > 0 && better(result, oi, sqd[pos - 1], idx[pos - 1])) {
        sqd[pos] = sqd[pos - 1]; idx[pos] = idx[pos - 1]; --pos;
      }
      sqd[pos] = result; idx[pos] = oi;
    }
    return;
  }
  const int f = nd.divfeat;
  const float val = q[f];
  const float diff1 = val - nd.divlow, diff2 = val - nd.divhigh;
  int best, other; float cut;
  if (diff1 + diff2 < 0) { best = nd.child1; other = nd.child2; cut = (val - nd.divhigh) * (val - nd.divhigh); }
  else { best = nd.child2; other = nd.child1; cut = (val - nd.divlow) * (val - nd.divlow); }
  search(best, q, mindistsq, dists, k, count, idx, sqd);
  const float dst = dists[f];
  const float md = mindistsq + cut - dst;
  dists[f] = cut;
  // `<=` so that equal-distance candidates with a smaller index are still found (tie rule above).  md is rounded differently
  // from a point's distance ((dx*dx + dy*dy) + dz*dz): for a point at the bound the two can differ by a few ulps, so the bound
  // gets a relative slack far above float rounding (a visit more costs time, never exactness)
  if (count < k || md <= sqd[k - 1] * (1.0f + 1e-4f)) search(other, q, md, dists, k, count, idx, sqd);
  dists[f] = dst;
}

int KdTree::knn(const float q[3], int k, int* idx, float* sqdist) const {
  if (root_ < 0 || k <= 0) return 0;
  float dists[3] = {0, 0, 0};
  float distsq = 0.f;
  for (int a = 0; a < 3; ++a) {
    if (q[a] < root_bbox_[2 * a]) { dists[a] = (q[a] - root_bbox_[2 * a]) * (q[a] - root_bbox_[2 * a]); distsq += dists[a]; }
    if (q[a] > root_bbox_[2 * a + 1]) { dists[a] = (q[a] - root_bbox_[2 * a + 1]) * (q[a] - root_bbox_[2 * a + 1]); distsq += dists[a]; }
  }
  int count = 0;
  search(root_, q, distsq, dists, k, count, idx, sqdist);
  return count;
}

}  // namespace orc
