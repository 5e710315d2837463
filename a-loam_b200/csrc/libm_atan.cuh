// The two transcendentals behind the reference's ring and sweep-walk decisions (scanRegistration.cpp:141-153,166,208-236),
// computed on the device so that they equal what an x86-64 build of the reference gets from the host's libm.
//
//   libm_atan2f      the float atan2 of glibc's flt-32 code (e_atan2f.c / s_atanf.c, the fdlibm algorithm) operation for
//                    operation.  It is not correctly rounded (it misses the nearest float on ~16 % of returns at lidar
//                    ranges) and CUDA's atan2f misses it differently, so neither a better nor a different atan2f would
//                    take the host's branch at an azimuth threshold of the walk.  Must be compiled without FMA contraction
//                    (-fmad=false on the device, -ffp-contract=off on the host), IEEE division, denormals kept.
//   elevation_deg    the float angle of :166, (float)(atan(d) * 180 / M_PI) with d = (double)z / sqrt((double)(x*x + y*y)).
//                    CUDA's double atan has up to 2 ulp of error; where that can move the double result across a float
//                    rounding boundary (it lies within kAngleBand double ulps of one), atan(d) is recomputed in
//                    double-double and rounded correctly, which is what glibc's atan returns on these arguments.  The
//                    host build runs the same test after libm's atan, so it models the device with a 0-ulp atan.
//
// Host-compilable (tests/cpp/libm_atan_check.cc builds it with g++ -ffp-contract=off to compare it with libm).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define LIBM_HD __host__ __device__ __forceinline__
#define LIBM_HD_NOINLINE static __host__ __device__ __noinline__   // internal linkage: several translation units include this header
#else
#define LIBM_HD inline
#define LIBM_HD_NOINLINE inline
#endif

namespace aloam {
namespace libm {

LIBM_HD float f_of(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f; memcpy(&f, &u, 4); return f;
#endif
}

LIBM_HD long long dbits_of(double f) {
#ifdef __CUDA_ARCH__
  return __double_as_longlong(f);
#else
  long long u; memcpy(&u, &f, 8); return u;
#endif
}

LIBM_HD double d_of(long long u) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(u);
#else
  double f; memcpy(&f, &u, 8); return f;
#endif
}

LIBM_HD int32_t bits_of(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_int(f);
#else
  int32_t u; memcpy(&u, &f, 4); return u;
#endif
}

// s_atanf.c: argument reduction to |x| < 7/16 around atan(0.5), atan(1), atan(1.5) or atan(inf), then an odd polynomial
// of degree 23 split into even and odd parts
LIBM_HD float atanf(float x) {
  const int32_t hx = bits_of(x), ix = hx & 0x7fffffff;
  int id;
  if (ix >= 0x4c000000) {                                      // |x| >= 2^25
    if (ix > 0x7f800000) return x + x;                         // NaN
    return hx > 0 ? f_of(0x3fc90fda) + f_of(0x33a22168) : -f_of(0x3fc90fda) - f_of(0x33a22168);
  }
  if (ix < 0x3ee00000) {                                       // |x| < 0.4375
    if (ix < 0x31000000) return x;                             // |x| < 2^-29
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {                                     // |x| < 1.1875
      if (ix < 0x3f300000) { id = 0; x = (2.0f * x - 1.0f) / (2.0f + x); }
      else { id = 1; x = (x - 1.0f) / (x + 1.0f); }
    } else if (ix < 0x401c0000) { id = 2; x = (x - 1.5f) / (1.0f + 1.5f * x); }   // |x| < 2.4375
    else { id = 3; x = -1.0f / x; }
  }
  const float z = x * x, w = z * z;
  const float s1 = z * (f_of(0x3eaaaaab) + w * (f_of(0x3e124925) + w * (f_of(0x3dba2e6e) + w * (f_of(0x3d886b35) +
                   w * (f_of(0x3d4bda59) + w * f_of(0x3c8569d7))))));
  const float s2 = w * (f_of(0xbe4ccccd) + w * (f_of(0xbde38e38) + w * (f_of(0xbd9d8795) + w * (f_of(0xbd6ef16b) +
                   w * f_of(0xbd15a221)))));
  if (id < 0) return x - x * (s1 + s2);
  float hi, lo;
  switch (id) {
    case 0: hi = f_of(0x3eed6338); lo = f_of(0x31ac3769); break;    // atan(0.5)
    case 1: hi = f_of(0x3f490fda); lo = f_of(0x33222168); break;    // atan(1)
    case 2: hi = f_of(0x3f7b985e); lo = f_of(0x33140fb4); break;    // atan(1.5)
    default: hi = f_of(0x3fc90fda); lo = f_of(0x33a22168); break;   // atan(inf)
  }
  const float r = hi - ((x * (s1 + s2) - lo) - x);
  return hx < 0 ? -r : r;
}

// e_atan2f.c
LIBM_HD float atan2f(float y, float x) {
  const float pi_o_4 = f_of(0x3f490fdb), pi_o_2 = f_of(0x3fc90fdb), pi = f_of(0x40490fdb), pi_lo = f_of(0xb3bbbd2e);
  const float tiny = 1.0e-30f;
  const int32_t hx = bits_of(x), ix = hx & 0x7fffffff, hy = bits_of(y), iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;      // NaN
  if (hx == 0x3f800000) return atanf(y);                     // x = 1
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);          // 2 * sign(x) + sign(y)
  if (iy == 0) {
    switch (m) {
      case 0: case 1: return y;
      case 2: return pi + tiny;
      default: return -pi - tiny;
    }
  }
  if (ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  if (ix == 0x7f800000) {
    if (iy == 0x7f800000) {
      switch (m) {
        case 0: return pi_o_4 + tiny;
        case 1: return -pi_o_4 - tiny;
        case 2: return 3.0f * pi_o_4 + tiny;
        default: return -3.0f * pi_o_4 - tiny;
      }
    }
    switch (m) {
      case 0: return 0.0f;
      case 1: return -0.0f;
      case 2: return pi + tiny;
      default: return -pi - tiny;
    }
  }
  if (iy == 0x7f800000) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  const int k = (iy - ix) >> 23;
  float z;
  if (k > 60) z = pi_o_2 + 0.5f * pi_lo;                      // |y / x| > 2^60
  else if (hx < 0 && k < -60) z = 0.0f;                       // |y| / x < -2^60
  else z = atanf(fabsf(y / x));
  switch (m) {
    case 0: return z;
    case 1: return -z;
    case 2: return pi - (z - pi_lo);
    default: return (z - pi_lo) - pi;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// double-double arithmetic (error-free transforms; fma for the exact product)
struct DD { double hi, lo; };

LIBM_HD DD two_sum(double a, double b) {
  const double s = a + b, bb = s - a;
  return {s, (a - (s - bb)) + (b - bb)};
}
LIBM_HD DD quick_two_sum(double a, double b) { const double s = a + b; return {s, b - (s - a)}; }
LIBM_HD DD dd_add(DD a, DD b) {
  DD s = two_sum(a.hi, b.hi);
  DD t = two_sum(a.lo, b.lo);
  s.lo += t.hi;
  s = quick_two_sum(s.hi, s.lo);
  s.lo += t.lo;
  return quick_two_sum(s.hi, s.lo);
}
LIBM_HD DD dd_mul(DD a, DD b) {
  const double p = a.hi * b.hi;
  double e = fma(a.hi, b.hi, -p);
  e += a.hi * b.lo + a.lo * b.hi;
  return quick_two_sum(p, e);
}
LIBM_HD DD dd_mul_d(DD a, double b) {
  const double p = a.hi * b;
  double e = fma(a.hi, b, -p);
  e += a.lo * b;
  return quick_two_sum(p, e);
}
LIBM_HD DD dd_div_d(DD a, double b) {
  const double q1 = a.hi / b;
  const double r = fma(-q1, b, a.hi) + a.lo;   // a - q1 b, exact in its leading part
  return quick_two_sum(q1, r / b);
}

// atan(d) rounded correctly to double, from an approximation a0 within a few ulps: one Newton step on tan in double-double,
//   atan(d) = a0 + atan((d cos a0 - sin a0) / (cos a0 + d sin a0)),
// with sin and cos of a0 (|a0| <= pi/2) from their Taylor series to 2^-106 and atan(delta) = delta (|delta| ~ 1e-15)
LIBM_HD_NOINLINE double atan_correct(double d, double a0) {
  const DD x2 = dd_mul({a0, 0.0}, {a0, 0.0});
  DD s = {a0, 0.0}, c = {1.0, 0.0}, ts = {a0, 0.0}, tc = {1.0, 0.0};
#pragma unroll 1
  for (int k = 1; k <= 16; ++k) {          // (pi/2)^33 / 33! < 2^-110
    ts = dd_div_d(dd_mul(ts, x2), -(double)((2 * k) * (2 * k + 1)));
    tc = dd_div_d(dd_mul(tc, x2), -(double)((2 * k - 1) * (2 * k)));
    s = dd_add(s, ts);
    c = dd_add(c, tc);
  }
  const DD num = dd_add(dd_mul_d(c, d), {-s.hi, -s.lo});
  const DD den = dd_add(c, dd_mul_d(s, d));
  const double delta = (num.hi + num.lo) / (den.hi + den.lo);
  return a0 + delta;
}

// double ulps around the double angle within which a float rounding boundary sends the return to atan_correct: the
// 2 ulp of CUDA's atan grow to at most ~9 ulp through * 180 and / M_PI
constexpr long long kAngleBand = 16;

// scanRegistration.cpp:166, float products, double sqrt / atan, * 180 / M_PI in double, stored to float
LIBM_HD float elevation_deg(float x, float y, float z) {
  constexpr double kPi = 3.14159265358979323846;  // M_PI
  const double d = (double)z / sqrt((double)(x * x + y * y));
  const double a = atan(d);
  const double t = a * 180.0 / kPi;
  const long long b = dbits_of(fabs(t));
  const float lo = (float)d_of(b > kAngleBand ? b - kAngleBand : 0), hi = (float)d_of(b + kAngleBand);
  if (lo != hi && t == t) return (float)(atan_correct(d, a) * 180.0 / kPi);
  return (float)t;
}

}  // namespace libm
}  // namespace aloam
