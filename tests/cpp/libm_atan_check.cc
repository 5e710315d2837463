// Host build of a-loam_b200/csrc/libm_atan.cuh for tests/libm_edge_cases.py: the device's atan2f restatement and its
// correctly rounded atan next to the host libm they stand for, and the exact search for float returns whose elevation
// lies on a float rounding boundary.  Compiled with -ffp-contract=off, as the kernels are with -fmad=false.  TEST
// INFRASTRUCTURE.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "libm_atan.cuh"

namespace L = aloam::libm;

static inline float f_of(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t u_of(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

extern "C" {

float lc_atan2f(float y, float x) { return L::atan2f(y, x); }
float lc_libm_atan2f(float y, float x) { return ::atan2f(y, x); }
double lc_atan_correct(double d, double a0) { return L::atan_correct(d, a0); }
float lc_elevation_deg(float x, float y, float z) { return L::elevation_deg(x, y, z); }

// restatement vs libm atan2f on n xorshift pairs: odd draws are any 64 bits (every class of float), even ones uniform in
// [-80, 80] m.  Returns the number of pairs whose bits differ (NaNs of either sign count as equal); the first at *first
static uint64_t g_s;
static inline uint64_t xr() { g_s ^= g_s << 13; g_s ^= g_s >> 7; g_s ^= g_s << 17; return g_s; }
long lc_compare_atan2f_random(long n, uint64_t seed, float* first) {
  g_s = seed | 1;
  long bad = 0;
  for (long i = 0; i < n; ++i) {
    float y, x;
    if (i & 1) { uint64_t r = xr(); y = f_of((uint32_t)r); x = f_of((uint32_t)(r >> 32)); }
    else {
      y = (float)((int64_t)(xr() >> 11) - (1ll << 52)) / (float)(1ll << 52) * 80.f;
      x = (float)((int64_t)(xr() >> 11) - (1ll << 52)) / (float)(1ll << 52) * 80.f;
    }
    const float a = ::atan2f(y, x), b = L::atan2f(y, x);
    if (u_of(a) != u_of(b) && !(isnan(a) && isnan(b))) { if (!bad) { first[0] = y; first[1] = x; } ++bad; }
  }
  return bad;
}

long lc_compare_atan2f_pairs(const float* y, const float* x, long n) {
  long bad = 0;
  for (long i = 0; i < n; ++i) bad += u_of(::atan2f(y[i], x[i])) != u_of(L::atan2f(y[i], x[i]));
  return bad;
}

// restatement vs libm atanf on every float with bits in [lo, hi) (NaN inputs skipped); the first mismatch at *first
long lc_compare_atanf_range(uint64_t lo, uint64_t hi, float* first) {
  long bad = 0;
  for (uint64_t u = lo; u < hi; ++u) {
    const float x = f_of((uint32_t)u);
    if (isnan(x)) continue;
    if (u_of(::atanf(x)) != u_of(L::atanf(x))) { if (!bad) *first = x; ++bad; }
  }
  return bad;
}

// float returns with (double)z / sqrt((double)h2) in [dlo, dhi]: h2 runs over every float with bits in [h2lo, h2hi), z over
// the float nearest to dmid * sqrt(h2) and its two neighbours.  Writes up to cap (z, h2) pairs (in no fixed order: the
// caller sorts them); returns how many exist
static long g_hits;
long lc_search_triples(double dlo, double dhi, double dmid, uint32_t h2lo, uint32_t h2hi, float* out, long cap) {
  long n = 0;
  g_hits = 0;
#pragma omp parallel for schedule(static) reduction(+ : n)
  for (uint32_t u = h2lo; u < h2hi; ++u) {
    const float h2 = f_of(u);
    const double s = sqrt((double)h2);
    const float zc = (float)(dmid * s);
    const float zs[3] = {zc, nextafterf(zc, -INFINITY), nextafterf(zc, INFINITY)};
    for (int k = 0; k < 3; ++k) {
      const double q = (double)zs[k] / s;
      if (q >= dlo && q <= dhi) {
        long slot;
#pragma omp atomic capture
        slot = g_hits++;
        if (slot < cap) { out[2 * slot] = zs[k]; out[2 * slot + 1] = h2; }
        ++n;
      }
    }
  }
  return n;
}

}  // extern "C"
