// The oracle of place recognition (include/aloam_b200.h, "place recognition"): the Scan Context descriptor of a scan, the column
// norms, the column-shifted distance, the ranking of a query's matches and the keyframe gate, restated from the header's
// definitions one operation at a time.  Built with -ffp-contract=off (oracle/place.mk): no product is contracted into an FMA.
// ORACLE = test infrastructure, like the rest of this directory.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {
constexpr int kRings = 20, kSectors = 60, kBins = kRings * kSectors;

// the total order of IEEE bit patterns (-0 < +0) as unsigned keys; 0 marks an empty bin
uint32_t ord_key(float v) {
  uint32_t b;
  std::memcpy(&b, &v, 4);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
float key_value(uint32_t k) {
  if (k == 0u) return 0.f;
  const uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float v;
  std::memcpy(&v, &b, 4);
  return v;
}
uint64_t ord_key64(double v) {
  uint64_t b;
  std::memcpy(&b, &v, 8);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
void norms(const float* d, double* n) {
  for (int c = 0; c < kSectors; ++c) {
    double s = 0.0;
    for (int r = 0; r < kRings; ++r) { const double v = d[r * kSectors + c]; s = s + v * v; }
    n[c] = std::sqrt(s);
  }
}
// D and the smallest shift reaching it, of query q (norms qn) against keyframe d (norms dn)
void distance(const float* q, const double* qn, const float* d, const double* dn, double* D, int* shift) {
  double best = 0.0;
  int bs = -1;
  for (int s = 0; s < kSectors; ++s) {
    double sim = 0.0;
    int cnt = 0;
    for (int c = 0; c < kSectors; ++c) {
      const int c2 = (c + s) % kSectors;
      if (qn[c] == 0.0 || dn[c2] == 0.0) continue;
      double dot = 0.0;
      for (int r = 0; r < kRings; ++r) dot = dot + (double)q[r * kSectors + c] * (double)d[r * kSectors + c2];
      sim = sim + dot / (qn[c] * dn[c2]);
      ++cnt;
    }
    const double dist = cnt ? 1.0 - sim / (double)cnt : 1.0;
    if (bs < 0 || dist < best) { best = dist; bs = s; }
  }
  *D = best;
  *shift = bs;
}
}  // namespace

extern "C" {

// the descriptor of clouds a (na points) then b (nb points), 4 floats per point
void orc_place_describe(const float* a, int na, const float* b, int nb, float max_range, float z_offset, float* desc) {
  std::vector<uint32_t> key(kBins, 0u);
  for (int i = 0; i < na + nb; ++i) {
    const float* p = i < na ? a + 4 * i : b + 4 * (i - na);
    const float x = p[0], y = p[1], z = p[2];
    const float r = std::sqrt(x * x + y * y);
    if (!(r < max_range)) continue;
    int ring = (int)((r * 20.0f) / max_range);
    if (ring > kRings - 1) ring = kRings - 1;
    float az = ::atan2f(y, x);
    if (az < 0.f) az = az + 6.28318548f;
    int sector = (int)((az * 60.0f) / 6.28318548f);
    if (sector > kSectors - 1) sector = kSectors - 1;
    const uint32_t k = ord_key(z + z_offset);
    uint32_t& slot = key[ring * kSectors + sector];
    if (k > slot) slot = k;
  }
  for (int i = 0; i < kBins; ++i) desc[i] = key_value(key[i]);
}

void orc_place_norms(const float* desc, double* norm) { norms(desc, norm); }

void orc_place_distance(const float* q, const float* d, double* D, int* shift) {
  double qn[kSectors], dn[kSectors];
  norms(q, qn);
  norms(d, dn);
  distance(q, qn, d, dn, D, shift);
}

// the k best of M keyframes (descriptor m at db + m * stride floats) for each of nq queries, ranked by (D, index): out n_q x k
void orc_place_query(const float* q, int nq, const float* db, long long stride, int M, int k, int* idx, int* shift, double* dist) {
  std::vector<double> dbn((size_t)M * kSectors);
  for (int m = 0; m < M; ++m) norms(db + (size_t)m * stride, &dbn[(size_t)m * kSectors]);
  std::vector<double> D(M);
  std::vector<int> S(M);
  for (int y = 0; y < nq; ++y) {
    const float* qy = q + (size_t)y * kBins;
    double qn[kSectors];
    norms(qy, qn);
    for (int m = 0; m < M; ++m) distance(qy, qn, db + (size_t)m * stride, &dbn[(size_t)m * kSectors], &D[m], &S[m]);
    uint64_t pk = 0;
    int pj = -1;
    for (int r = 0; r < k; ++r) {
      uint64_t bk = 0;
      int bj = -1;
      for (int m = 0; m < M; ++m) {
        const uint64_t km = ord_key64(D[m]);
        if (pj >= 0 && !(pk < km || (pk == km && pj < m))) continue;
        if (bj < 0 || km < bk) { bk = km; bj = m; }
      }
      idx[y * k + r] = bj;
      shift[y * k + r] = bj >= 0 ? S[bj] : -1;
      dist[y * k + r] = bj >= 0 ? D[bj] : -1.0;
      pk = bk; pj = bj;
    }
  }
}

// the keyframe gate: 1 when a lane whose last keyframe has map translation last_t (NULL: an empty table) takes a row at map
// translation t, with keyframe_gap^2 = gap2
int orc_place_gate(const double* last_t, const double* t, double gap2) {
  if (!last_t) return 1;
  const double dx = t[0] - last_t[0], dy = t[1] - last_t[1], dz = t[2] - last_t[2];
  return (dx * dx + dy * dy) + dz * dz >= gap2;
}

}  // extern "C"
