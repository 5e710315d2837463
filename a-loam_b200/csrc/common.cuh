// Shared device/host definitions for the sm_90a kernels.  Everything in csrc/ is compiled with -fmad=false:
// the reference is an x86-64 baseline build (CMakeLists.txt:4-6, no -march => no FMA), and the discrete decisions
// of the hot path (feature picks, nearest neighbours, voxel indices) depend on float32 results bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#define ALOAM_WARP 32

struct __align__(16) Pt4 { float x, y, z, i; };  // pcl::PointXYZI payload (common.h:43)

// per-context scalars that live in device memory (written by kernels, read by later kernels; never by the
// host inside the per-scan pipeline)
struct ScanScalars {
  int first_valid;   // first raw index that survives NaN / minimum-range removal (scanRegistration.cpp:136-137)
  int last_valid;    // last such index
  int half_idx;      // raw index of the return that flips halfPassed (scanRegistration.cpp:220-223), INT_MAX if none
  int n_full;        // points in the ring-major cloud (cloudSize after :243)
  float start_ori;   // :141
  float end_ori;     // :142-153
  int error;         // sticky device-side error code (ring too large, ...)
  int pad;
};

// feature cloud set produced by one scan (device resident)
struct FeatureCounts {
  int n_sharp, n_less_sharp, n_flat, n_less_flat;
};

// programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become
// resident before its predecessor in the stream has finished. pdl_wait() blocks until the predecessor grid has completed
// and its memory is visible (a no-op for a normal launch); pdl_launch_dependents() lets the successor start launching.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

#define CUDA_CHECK_RET(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      fprintf(stderr, "[aloam_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
              cudaGetErrorString(_e));                                                         \
      return ALOAM_ERR_CUDA;                                                                   \
    }                                                                                          \
  } while (0)

#ifdef __CUDACC__
__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }

// (d2, idx) lexicographic warp arg-min; d2 >= 0 so its bit pattern orders like the float
__device__ __forceinline__ void warp_argmin(float& d2, int& idx) {
  unsigned bits = __float_as_uint(d2);
  unsigned mb = __reduce_min_sync(0xffffffffu, bits);
  unsigned cand = (bits == mb) ? (unsigned)idx : 0xffffffffu;
  unsigned mi = __reduce_min_sync(0xffffffffu, cand);
  d2 = __uint_as_float(mb);
  idx = (int)mi;
}

// Eigen QuaternionBase::slerp(s, q) called on the identity (laserOdometry.cpp:120, lidarFactor.hpp:29-30,81-82): double
// precision, (x, y, z, w).  |q.w| >= 1 - eps takes the linear blend, q.w < 0 flips the second weight; slerp(1, q) == q exactly.
__device__ __forceinline__ void slerp_identity(const double* q, double s, double* o) {
  const double one = 1.0 - 2.220446049250313e-16;
  const double d = q[3], ad = fabs(d);
  double w0, w1;
  if (ad >= one) { w0 = 1.0 - s; w1 = s; }
  else {
    const double th = acos(ad), sth = sin(th);
    w0 = sin((1.0 - s) * th) / sth;
    w1 = sin(s * th) / sth;
  }
  if (d < 0.0) w1 = -w1;
  o[0] = w1 * q[0]; o[1] = w1 * q[1]; o[2] = w1 * q[2]; o[3] = w0 + w1 * q[3];
}

__device__ __forceinline__ float sqdist3(float ax, float ay, float az, float bx, float by, float bz) {
  // ((dx*dx) + dy*dy) + dz*dz in float, no contraction (compiled with -fmad=false)
  float dx = ax - bx, dy = ay - by, dz = az - bz;
  return dx * dx + dy * dy + dz * dz;
}
#endif
