// Device-resident Levenberg-Marquardt -- replaces the ceres::Solve calls at laserOdometry.cpp:494-499 and
// laserMapping.cpp:712-720 together with the residual functors of lidarFactor.hpp (:12-55 edge, :57-104 plane,
// :106-138 plane-norm) and everything Ceres drives around them (AutoDiff Jacobians, HuberLoss(0.1) + Corrector,
// EigenQuaternionParameterization, trust-region loop, DENSE_QR step).
//
// Shape: the whole solve is ONE launch of ONE thread-block cluster (8 CTAs x 288 threads, co-scheduled on one
// GPC) and never returns to the host.  Each pass evaluates every residual block with the closed-form tangent
// Jacobian (SURVEY.md 8a "Residual math") and reduces the 28 numbers the 6-dof problem boils down to -- upper
// triangle of J^T J (21), J^T r (6), cost (1) -- plus the two block counts:
//     thread  -> warp   : transpose through shared memory, lane L adds column L in a fixed tree
//     warp    -> CTA    : warp 0 adds the 9 partial vectors in a fixed tree
//     CTA     -> cluster: every CTA PUSHES its vector into the shared memory of all 8 CTAs (distributed shared memory
//                         stores), one cluster barrier, then adds the 8 vectors in rank order, so all CTAs hold
//                         bit-identical totals (double-buffered by pass parity).
// No float atomics anywhere => run-to-run deterministic.  Thread 0 of every CTA then takes the SAME trust-region
// decision redundantly (no broadcast step), exactly as Ceres' TrustRegionMinimizer / LevenbergMarquardtStrategy:
//   Jacobi scaling 1/(1+||J_j||) fixed at iteration 0, D^2 = clamp(diag(Js^T Js), 1e-6, 1e32) (re-used after a
//   rejected step), (Js^T Js + D^2/radius) y = Js^T r  [normal-equation form of Ceres' QR on [Js; sqrt(D^2/radius)]],
//   model_cost_change, Plus(), parameter / function tolerance tests, rho > 1e-3 accept with
//   radius / max(1/3, 1-(2 rho-1)^3), reject with radius / decrease_factor, decrease_factor *= 2.
// The candidate evaluation already carries J^T J and J^T r, so an accepted step needs no second pass (Ceres
// evaluates cost-only, then re-evaluates with Jacobians): <= 1 + max_iters passes per solve instead of <= 1 + 2 max_iters.
//
// This file is compiled WITH fused multiply-add (the only one): the solve is double precision and is compared to the
// oracle at 1e-9, not bit for bit; the float32 decisions that must be bit-exact live in features.cu / odometry.cu.
#include <cfloat>
#include <cooperative_groups.h>
#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace aloam {

namespace {

constexpr int NT = ALOAM_LM_THREADS;
constexpr int NW = NT / 32;

struct V3 { double x, y, z; };
__device__ __forceinline__ V3 crossd(const V3& a, const V3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

// acc layout: [0..20] upper triangle of J^T J row-major (00,01,..05,11,..,55), [21..26] J^T r, [27] cost
__device__ __forceinline__ void accumulate_row(double* acc, const double j[6], double r) {
  int k = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
#pragma unroll
    for (int b = a; b < 6; ++b) acc[k++] += j[a] * j[b];
  }
#pragma unroll
  for (int a = 0; a < 6; ++a) acc[21 + a] += j[a] * r;
}

__device__ __forceinline__ void huber_rho(double huber_a, double sq, double& rho0, double& sr) {
  const double bb = huber_a * huber_a;
  if (sq > bb) {
    const double irr = rsqrt(sq), rr = sq * irr;
    rho0 = 2.0 * huber_a * rr - bb;
    sr = sqrt(fmax(DBL_MIN, huber_a * irr));   // Corrector: rho'' <= 0 => scale residual and Jacobian by sqrt(rho')
  } else {
    rho0 = sq; sr = 1.0;
  }
}

// General interpolation ratio s != 1 (DISTORTION build, lidarFactor.hpp:27-33,79-85): lp = slerp(I, q, s) p + s t.
// With Ceres' left-multiplicative Plus, a perturbation eps = 2 dtheta of q moves q^s by the left perturbation M eps,
// M = s Jl(s phi) Jl(phi)^-1 (phi = rotation vector of q, Jl = left Jacobian of SO(3)), a polynomial m0 I + m1 K + m2 K^2 in
// K = [phi / |phi|]x.  Row of a residual with gradient g wrt lp:  [ (2 (Rp x g))^T M , s g^T ].  The same closed form as
// include/lidarFactor.hpp (checked there against Jet autodiff of the literal functor); M = I for s = 1.
struct StartFrame {
  V3 Rp;             // R^s p
  V3 k;              // rotation axis
  double m0, m1, m2, s;
};
__device__ __noinline__ void start_frame_general(const double* x, const V3& cp, double s, StartFrame& F) {
  double qs[4];
  slerp_identity(x, s, qs);
  const V3 u{qs[0], qs[1], qs[2]};
  V3 uv = crossd(u, cp);
  uv.x += uv.x; uv.y += uv.y; uv.z += uv.z;
  const V3 c2 = crossd(u, uv);
  F.Rp = V3{cp.x + qs[3] * uv.x + c2.x, cp.y + qs[3] * uv.y + c2.y, cp.z + qs[3] * uv.z + c2.z};
  F.s = s;
  const double sgn = x[3] < 0.0 ? -1.0 : 1.0;
  const double vx = sgn * x[0], vy = sgn * x[1], vz = sgn * x[2], w = sgn * x[3];
  const double vn = sqrt(vx * vx + vy * vy + vz * vz);
  if (vn < 1e-12) { F.k = V3{1.0, 0.0, 0.0}; F.m0 = s; F.m1 = 0.0; F.m2 = 0.0; return; }
  const double th = 2.0 * atan2(vn, w);
  F.k = V3{vx / vn, vy / vn, vz / vn};
  const double uang = s * th;
  const double a1 = fabs(uang) < 1e-8 ? 0.5 * uang : (1.0 - cos(uang)) / uang;
  const double a2 = fabs(uang) < 1e-4 ? uang * uang / 6.0 : 1.0 - sin(uang) / uang;
  const double b1 = -0.5 * th;
  const double b2 = 1.0 - 0.5 * th * cos(0.5 * th) / sin(0.5 * th);
  F.m0 = s;
  F.m1 = s * (b1 + a1 - a1 * b2 - a2 * b1);
  F.m2 = s * (b2 + a2 + a1 * b1 - a2 * b2);
}
// Jacobian row for gradient g wrt lp, scaled by sr
template <bool GENERAL>
__device__ __forceinline__ void start_row(const StartFrame& F, const V3& g, double sr, double* j) {
  const V3 t = crossd(F.Rp, g);
  V3 h{2.0 * t.x, 2.0 * t.y, 2.0 * t.z};
  if (GENERAL && (F.m1 != 0.0 || F.m2 != 0.0 || F.m0 != 1.0)) {
    const V3 hk = crossd(h, F.k), hkk = crossd(hk, F.k);
    h = V3{F.m0 * h.x + F.m1 * hk.x + F.m2 * hkk.x, F.m0 * h.y + F.m1 * hk.y + F.m2 * hkk.y, F.m0 * h.z + F.m1 * hk.z + F.m2 * hkk.z};
  }
  j[0] = h.x * sr; j[1] = h.y * sr; j[2] = h.z * sr;
  j[3] = F.s * g.x * sr; j[4] = F.s * g.y * sr; j[5] = F.s * g.z * sr;
}

// GENERAL = false: every block has s == 1 (the reference build: DISTORTION 0 odometry, all scan-to-map blocks); the slerp path
// is not even compiled in, which keeps the common kernel at its round-1 register budget and code size.
template <bool GENERAL>
__device__ __forceinline__ void eval_block(const BlockRec& rb, const double* x, double huber_a, double* acc) {
  // lp = R(q)^s cp + s t   (s == 1 for every block the reference build makes: slerp(1, q) == q)
  const V3 cp{rb.cp[0], rb.cp[1], rb.cp[2]};
  StartFrame F;
  const double s = (!GENERAL || rb.type == 2) ? 1.0 : rb.s;
  if (!GENERAL || s == 1.0) {
    const V3 u{x[0], x[1], x[2]};
    const double w = x[3];
    V3 uv = crossd(u, cp);
    uv.x += uv.x; uv.y += uv.y; uv.z += uv.z;
    const V3 c2 = crossd(u, uv);
    F.Rp = V3{cp.x + w * uv.x + c2.x, cp.y + w * uv.y + c2.y, cp.z + w * uv.z + c2.z};
    F.k = V3{1.0, 0.0, 0.0}; F.m0 = 1.0; F.m1 = 0.0; F.m2 = 0.0; F.s = 1.0;
  } else {
    StartFrame G;                       // out of line and through its own stack copy: the de-skew path must neither grow the
    start_frame_general(x, cp, s, G);   // common path's code nor force F into local memory
    F = G;
  }
  const V3 lp{F.Rp.x + s * x[4], F.Rp.y + s * x[5], F.Rp.z + s * x[6]};
  // d lp / d dtheta = -2 [Rp]x M  (Ceres Plus is delta_q (x) q with a half-angle delta) ; d lp / d t = s I
  // row of J for a residual with gradient n wrt lp:  [ (2 (Rp x n))^T M , s n^T ]
  if (rb.type == 0) {
    const V3 a{rb.a[0], rb.a[1], rb.a[2]}, b{rb.b[0], rb.b[1], rb.b[2]};
    const V3 la{lp.x - a.x, lp.y - a.y, lp.z - a.z}, lb{lp.x - b.x, lp.y - b.y, lp.z - b.z};
    const V3 nu = crossd(la, lb);
    const double idn = rb.w;  // 1 / |a - b|
    const double r[3] = {nu.x * idn, nu.y * idn, nu.z * idn};
    const V3 wv{(b.x - a.x) * idn, (b.y - a.y) * idn, (b.z - a.z) * idn};
    // d r / d lp = [wv]x ; rows: n0 = (0,-wz,wy), n1 = (wz,0,-wx), n2 = (-wy,wx,0)
    const V3 ns[3] = {V3{0.0, -wv.z, wv.y}, V3{wv.z, 0.0, -wv.x}, V3{-wv.y, wv.x, 0.0}};
    double rho0, sr;
    huber_rho(huber_a, r[0] * r[0] + r[1] * r[1] + r[2] * r[2], rho0, sr);
    acc[27] += 0.5 * rho0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double j[6];
      start_row<GENERAL>(F, ns[k], sr, j);
      accumulate_row(acc, j, r[k] * sr);
    }
  } else {
    V3 n; double r;
    if (rb.type == 1) {
      n = V3{rb.b[0], rb.b[1], rb.b[2]};
      r = (lp.x - rb.a[0]) * n.x + (lp.y - rb.a[1]) * n.y + (lp.z - rb.a[2]) * n.z;
    } else {
      n = V3{rb.a[0], rb.a[1], rb.a[2]};
      r = n.x * lp.x + n.y * lp.y + n.z * lp.z + rb.s;
    }
    double rho0, sr;
    huber_rho(huber_a, r * r, rho0, sr);
    acc[27] += 0.5 * rho0;
    double j[6];
    start_row<GENERAL>(F, n, sr, j);
    accumulate_row(acc, j, r * sr);
  }
}

// 32 values per lane -> lane L holds the warp total of value L (fixed summation tree)
__device__ __forceinline__ double warp_transpose_reduce(double (&v)[32]) {
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    const bool upper = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const double send = upper ? v[i] : v[i + half];
      const double keep = upper ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
  return v[0];
}

// sin(n)/n and cos(n).  LM steps are small rotations: below 0.25 rad both are evaluated as Taylor polynomials in n^2
// (truncation < 1e-17 relative, i.e. the same <= 1 ulp class as libm's sin / cos) -- 16 FMAs instead of two libm calls
// and a division on the serial trust-region path; larger angles take the libm route.
__device__ __forceinline__ void sinc_cos(double n, double& sinc, double& c) {
  if (n < 0.25) {
    const double t = n * n;
    double p = -1.0 / 6227020800.0;                 // sin(n)/n = 1 - t/3! + t^2/5! - ... - t^6/13!
    p = fma(p, t, 1.0 / 39916800.0);
    p = fma(p, t, -1.0 / 362880.0);
    p = fma(p, t, 1.0 / 5040.0);
    p = fma(p, t, -1.0 / 120.0);
    p = fma(p, t, 1.0 / 6.0);
    sinc = fma(-p, t, 1.0);
    double q = 1.0 / 87178291200.0;                 // cos(n) = 1 - t/2! + t^2/4! - ... + t^7/14!
    q = fma(q, t, -1.0 / 479001600.0);
    q = fma(q, t, 1.0 / 3628800.0);
    q = fma(q, t, -1.0 / 40320.0);
    q = fma(q, t, 1.0 / 720.0);
    q = fma(q, t, -1.0 / 24.0);
    q = fma(q, t, 0.5);
    c = fma(-q, t, 1.0);
  } else {
    sinc = sin(n) / n;
    c = cos(n);
  }
}

// ceres::EigenQuaternionParameterization::Plus + plain addition on t
__device__ __forceinline__ void plus7(const double* x, const double* d, double* o) {
  const double n = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (n > 0.0) {
    double s, aw;
    sinc_cos(n, s, aw);
    const double ax = s * d[0], ay = s * d[1], az = s * d[2];
    const double bx = x[0], by = x[1], bz = x[2], bw = x[3];
    o[3] = aw * bw - ax * bx - ay * by - az * bz;
    o[0] = aw * bx + ax * bw + ay * bz - az * by;
    o[1] = aw * by + ay * bw + az * bx - ax * bz;
    o[2] = aw * bz + az * bw + ax * by - ay * bx;
  } else {
    o[0] = x[0]; o[1] = x[1]; o[2] = x[2]; o[3] = x[3];
  }
  o[4] = x[4] + d[3]; o[5] = x[5] + d[4]; o[6] = x[6] + d[5];
}

// trust-region state of one solve (thread 0 only).  Shared memory in k_lm_solve, global memory in the sharded path.
// The accepted point's reduced totals (packed: 21 upper-triangle J^T J, 6 J^T r, cost) are NOT copied into the state on
// the cluster path: the kernel double-buffers its totals and `acc_buf` says which buffer belongs to the accepted point;
// the sharded path keeps them in `acc`.
struct TrState {
  double x[7], xc[7], acc[28], scale[6], diag[6];
  double cost, radius, decrease_factor, mcc, gmax, x_norm;
  int reuse_diag, last_successful, iteration, num_invalid, num_successful, num_evals, termination, trace_rows;
  int go;       // 1: xc holds a candidate that must be evaluated next ; 0: the solve is over
  int acc_buf;  // cluster path: index of the totals buffer of the accepted point
  int n_res;
};

// max-norm of Plus(x, -g) - x.  The translation part is |g_t| exactly; the quaternion part (sin / cos / sqrt in double)
// is only evaluated when it can change the `<= tol` decision, i.e. when the translation part is already <= tol.
__device__ __forceinline__ double gradient_max(const double* x, const double* g, double tol) {
  const double mt = fmax(fmax(fabs(g[3]), fabs(g[4])), fabs(g[5]));
  if (mt > tol) return mt;
  double ng[6], xp[7];
#pragma unroll
  for (int k = 0; k < 6; ++k) ng[k] = -g[k];
  plus7(x, ng, xp);
  double m = 0;
#pragma unroll
  for (int k = 0; k < 7; ++k) m = fmax(m, fabs(xp[k] - x[k]));
  return m;
}

// packed index of J^T J entry (a, c), a <= c
__device__ __forceinline__ constexpr int pk(int a, int c) { return a * 6 - (a * (a - 1)) / 2 + (c - a); }

// (Hs + diag/radius) y = b by Cholesky ; only the lower triangle Hs[i][j], i >= j, is read ; returns false on breakdown
__device__ __forceinline__ bool chol_solve6(const double (&Hs)[6][6], const double* dr, const double* b, double* y) {
  // L holds the strict lower triangle, inv[j] = 1 / L[j][j]  (one rsqrt per column, no divisions).  Every dot product
  // ends with its most recently produced operand, so the dependent chain per column is one FMA + rsqrt + one multiply.
  double L[6][6], inv[6], z[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double d = Hs[j][j] + dr[j];
    double zj = b[j];
#pragma unroll
    for (int k = 0; k < 6; ++k) if (k < j) { d -= L[j][k] * L[j][k]; zj -= L[j][k] * z[k]; }
    if (!(d > 0.0)) return false;
    inv[j] = rsqrt(d);
    z[j] = zj * inv[j];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      if (i > j) {
        double s = Hs[i][j];
#pragma unroll
        for (int k = 0; k < 6; ++k) if (k < j) s -= L[i][k] * L[j][k];
        L[i][j] = s * inv[j];
      }
    }
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double s = z[i];
#pragma unroll
    for (int k = 5; k >= 0; --k) if (k > i) s -= L[k][i] * y[k];   // descending: y[i + 1], the newest, comes last
    y[i] = s * inv[i];
  }
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) ok = ok && isfinite(y[i]);
  return ok;
}

// `trace` = where the rows go: a shared-memory staging array in the cluster kernel (flushed once by tr_finish: a store through the
// generic `summary` pointer in the middle of the step would force the compiler to re-read everything it holds from shared memory),
// summary->trace itself in the sharded path
__device__ __forceinline__ void tr_trace(TrState& T, double (*trace)[8], bool writer, double c, double cc, double gm, double sn,
                                         double rd, double rad, int valid, int succ) {
  if (T.trace_rows < ALOAM_LM_MAX_TRACE) {
    if (writer) {
      double* o = trace[T.trace_rows];
      o[0] = c; o[1] = cc; o[2] = gm; o[3] = sn; o[4] = rd; o[5] = rad; o[6] = valid; o[7] = succ;
    }
    ++T.trace_rows;
  }
}

// produce the next candidate (-> T.xc, T.go = 1) or stop (T.go = 0).  A = packed totals of the accepted point.
__device__ __forceinline__ void tr_next_candidate(TrState& T, const double* A, const LmParams& prm, double (*trace)[8], bool writer) {
  double sc[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) sc[j] = T.scale[j];
  for (;;) {
    if (T.iteration >= prm.max_iters) { T.termination = 0; T.go = 0; return; }
    if (T.last_successful && T.gmax <= prm.gradient_tolerance) { T.termination = 1; T.go = 0; return; }
    if (T.radius < prm.min_radius) { T.termination = 5; T.go = 0; return; }
    ++T.iteration;
    T.last_successful = 0;
    if (!T.reuse_diag) {
#pragma unroll
      for (int j = 0; j < 6; ++j) T.diag[j] = fmin(fmax(sc[j] * sc[j] * A[pk(j, j)], prm.min_lm_diagonal), prm.max_lm_diagonal);
    }
    double Hs[6][6], b[6], y[6], dr[6];
    const double ir = 1.0 / T.radius;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int c = 0; c < 6; ++c) if (c <= a) Hs[a][c] = sc[c] * A[pk(c, a)] * sc[a];
      b[a] = sc[a] * A[21 + a];
      dr[a] = T.diag[a] * ir;
    }
    const bool ok = chol_solve6(Hs, dr, b, y);
    T.reuse_diag = 1;
    double mcc = 0;
    if (ok) {
      // model_cost_change = -(Js step)^T (r + Js step / 2) = y^T b - 1/2 y^T Hs y  with step = -y.  Since
      // (Hs + D/radius) y = b :  y^T Hs y = y^T b - sum (D/radius)_a y_a^2 , hence
      // model_cost_change = 1/2 (y^T b + sum (D/radius)_a y_a^2)  -- 12 FMAs instead of a 6x6 matrix-vector product
      double yb = 0, ydy = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) { yb += y[a] * b[a]; ydy += dr[a] * y[a] * y[a]; }
      mcc = 0.5 * (yb + ydy);
    }
    T.mcc = mcc;
    if (!(ok && mcc > 0.0)) {  // invalid step
      if (++T.num_invalid >= prm.max_invalid) { tr_trace(T, trace, writer, T.cost, 0, T.gmax, 0, 0, T.radius, 0, 0); T.termination = 5; T.go = 0; return; }
      T.radius *= 0.5;
      tr_trace(T, trace, writer, T.cost, 0, T.gmax, 0, 0, T.radius, 0, 0);
      continue;
    }
    T.num_invalid = 0;
    double delta[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) delta[k] = -y[k] * sc[k];
    plus7(T.x, delta, T.xc);
    T.go = 1;
    return;
  }
}

// iteration 0: totals of the evaluation at x ; tot[28], tot[29] = number of edge / plane blocks
// Returns true when the caller has to produce the first candidate (tr_next_candidate on the same totals): the big step routine
// has ONE call site per kernel, shared with tr_after_eval.
__device__ __forceinline__ bool tr_start(TrState& T, const double* x, const double* tot, const LmParams& prm, LmSummary* summary, bool summary_writer,
                                         double (*trace)[8], bool writer) {
  const int ne = (int)(tot[28] + 0.5), np = (int)(tot[29] + 0.5);
#pragma unroll
  for (int k = 0; k < 7; ++k) { T.x[k] = x[k]; T.xc[k] = x[k]; }
  T.cost = tot[27];
  T.radius = prm.initial_radius; T.decrease_factor = 2.0; T.mcc = 0; T.gmax = 0;
  T.reuse_diag = 0; T.last_successful = 0; T.iteration = 0; T.num_invalid = 0; T.num_successful = 0; T.num_evals = 1;
  T.termination = 0; T.trace_rows = 0; T.n_res = ne + np; T.go = 0; T.acc_buf = 0; T.x_norm = 0;
#pragma unroll
  for (int j = 0; j < 6; ++j) { T.scale[j] = 0; T.diag[j] = 0; }
  if (summary_writer) { summary->initial_cost = T.cost; summary->n_edge = ne; summary->n_plane = np; }
  if (ne + np == 0) { T.termination = 4; return false; }  // Ceres: nothing to optimise, parameters untouched
#pragma unroll
  for (int j = 0; j < 6; ++j) T.scale[j] = 1.0 / (1.0 + sqrt(tot[pk(j, j)]));
  T.gmax = gradient_max(T.x, tot + 21, prm.gradient_tolerance);
  double xn = 0;
#pragma unroll
  for (int k = 0; k < 7; ++k) xn += T.x[k] * T.x[k];
  T.x_norm = sqrt(xn);
  tr_trace(T, trace, writer, T.cost, 0, T.gmax, 0, 0, T.radius, 0, 0);
  if (T.gmax <= prm.gradient_tolerance) { T.termination = 1; return false; }
  return true;
}

// after the evaluation of candidate T.xc (totals `tot`; `A` = totals of the currently accepted point): tolerance tests,
// accept / reject.  Returns 0 when the solve is over, 1 when the candidate was rejected, 2 when it was accepted (its totals are the
// accepted ones now); for 1 and 2 the caller produces the next candidate.
__device__ __forceinline__ int tr_after_eval(TrState& T, const double* tot, const LmParams& prm, double (*trace)[8], bool writer) {
  ++T.num_evals;
  const double cand_cost = tot[27];
  // Every long-latency operation of the step (two square roots, three divisions) is issued up front, before the branches that
  // decide which of them are used: they are independent of each other except radius_acc <- rho, so one thread overlaps their
  // latencies instead of paying them one after the other.  Each value is exactly the one the branch would have computed.
  double sn2 = 0, xn2 = 0;
#pragma unroll
  for (int k = 0; k < 7; ++k) { sn2 += (T.x[k] - T.xc[k]) * (T.x[k] - T.xc[k]); xn2 += T.xc[k] * T.xc[k]; }
  const double sn = sqrt(sn2);
  const double xn_cand = sqrt(xn2);                          // |xc|: the new x_norm if the step is accepted
  const double cost_change = T.cost - cand_cost;
  const double rho = cost_change / T.mcc;                    // mcc > 0 for every candidate that was evaluated
  const double radius_rej = T.radius / T.decrease_factor;
  const double tq = 2.0 * rho - 1.0;
  const double radius_acc = fmin(prm.max_radius, T.radius / fmax(1.0 / 3.0, 1.0 - tq * tq * tq));
  if (sn <= prm.parameter_tolerance * (T.x_norm + prm.parameter_tolerance)) {
    tr_trace(T, trace, writer, T.cost, 0, T.gmax, sn, 0, T.radius, 1, 0); T.termination = 2; T.go = 0; return 0;
  }
  if (fabs(cost_change) <= prm.function_tolerance * T.cost) {
    tr_trace(T, trace, writer, T.cost, cost_change, T.gmax, sn, 0, T.radius, 1, 0); T.termination = 3; T.go = 0; return 0;
  }
  const bool accept = rho > prm.min_relative_decrease;
  if (accept) {
#pragma unroll
    for (int k = 0; k < 7; ++k) T.x[k] = T.xc[k];
    T.x_norm = xn_cand;
    T.cost = cand_cost;
    T.gmax = gradient_max(T.x, tot + 21, prm.gradient_tolerance);
    T.last_successful = 1;
    ++T.num_successful;
    T.radius = radius_acc;
    T.decrease_factor = 2.0;
    T.reuse_diag = 0;
    tr_trace(T, trace, writer, T.cost, cost_change, T.gmax, sn, rho, T.radius, 1, 1);
  } else {
    T.radius = radius_rej;
    T.decrease_factor *= 2.0;
    T.reuse_diag = 1;
    tr_trace(T, trace, writer, T.cost, cost_change, T.gmax, sn, rho, T.radius, 1, 0);
  }
  return accept ? 2 : 1;
}

// the part of the state the step works on, between its home (shared / global memory) and a local copy that lives in registers
// for the duration of a step (`acc`, the sharded path's totals, stays where it is)
__device__ __forceinline__ void tr_copy(TrState& d, const TrState& s) {
#pragma unroll
  for (int k = 0; k < 7; ++k) { d.x[k] = s.x[k]; d.xc[k] = s.xc[k]; }
#pragma unroll
  for (int k = 0; k < 6; ++k) { d.scale[k] = s.scale[k]; d.diag[k] = s.diag[k]; }
  d.cost = s.cost; d.radius = s.radius; d.decrease_factor = s.decrease_factor; d.mcc = s.mcc; d.gmax = s.gmax; d.x_norm = s.x_norm;
  d.reuse_diag = s.reuse_diag; d.last_successful = s.last_successful; d.iteration = s.iteration; d.num_invalid = s.num_invalid;
  d.num_successful = s.num_successful; d.num_evals = s.num_evals; d.termination = s.termination; d.trace_rows = s.trace_rows;
  d.go = s.go; d.acc_buf = s.acc_buf; d.n_res = s.n_res;
}

__device__ void tr_finish(const TrState& T, double* x7, LmSummary* summary, const double (*staged_trace)[8] = nullptr) {
#pragma unroll
  for (int k = 0; k < 7; ++k) x7[k] = T.x[k];
  if (staged_trace)
    for (int r = 0; r < T.trace_rows && r < ALOAM_LM_MAX_TRACE; ++r)
      for (int k = 0; k < 8; ++k) summary->trace[r][k] = staged_trace[r][k];
  summary->termination = T.termination;
  summary->num_iterations = T.iteration;
  summary->num_successful = T.num_successful;
  summary->num_jac_evals = T.num_evals;
  summary->final_cost = T.cost;
  summary->trace_rows = T.trace_rows;
}

// every thread of the cluster evaluates its share of the blocks at x ; afterwards s_tot[0..29] (written and read by warp 0
// only) holds the cluster-wide totals in every CTA (slots 28 / 29 = edge / plane block counts).
//   thread -> warp : the 30 accumulators are transposed through shared memory (15 STS.128 per thread, then lane L adds
//                    column L of its warp's 32 rows in a fixed order) -- 80 instructions instead of the 217 of a
//                    select + shuffle butterfly in double precision
//   warp -> CTA    : warp 0 adds the NW partial vectors
//   CTA -> cluster : warp 0 PUSHES its vector into every CTA's shared memory (DSMEM stores), one cluster barrier, then
//                    every CTA adds the 8 vectors it received in rank order => bit-identical totals everywhere.
// `rb0` is this thread's first block, kept in registers across the passes of a solve.
// Block b of a pass is evaluated by the thread with first_block_index == b mod (cluster threads).  Consecutive 32-block
// chunks go round-robin over the CTAs (chunk c -> CTA c mod 8, warp c / 8): the association kernels write all edge
// blocks first (3 residual rows each, ~2x the work of a plane block) and leave the unused slots at the end of each
// section, so a CTA-major assignment would give three CTAs all the edges and the last CTAs nothing.
__device__ __forceinline__ int first_block_index(unsigned crank, unsigned csize) {
  return (int)(((threadIdx.x >> 5) * csize + crank) * 32u + (threadIdx.x & 31u));
}

constexpr int RS = 30;   // doubles per thread row of the transpose scratch (240 B: 16-byte aligned, bank-conflict free)
template <bool GENERAL, typename Cluster>
__device__ __forceinline__ void cluster_evaluate(Cluster& cluster, const BlockRec* __restrict__ blocks, int n, const BlockRec& rb0,
                                                 const double* xs, double huber_a, double* s_red, double (*s_part)[32],
                                                 double (*s_in)[8][32], double* s_tot, int& pass, long long& cyc_blocks, long long& cyc_barrier) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long t_a = clock64();
  const unsigned crank = cluster.block_rank(), csize = cluster.num_blocks();
  const int gtid = first_block_index(crank, csize), gstride = (int)csize * NT;
  double x[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) x[k] = xs[k];
  double acc[RS];
#pragma unroll
  for (int k = 0; k < RS; ++k) acc[k] = 0.0;
  if (gtid < n) {
    BlockRec rb = rb0;
    for (int b = gtid;;) {
      if (rb.type >= 0) {
        eval_block<GENERAL>(rb, x, huber_a, acc);
        acc[28] += (rb.type == 0) ? 1.0 : 0.0;
        acc[29] += (rb.type > 0) ? 1.0 : 0.0;
      }
      b += gstride;
      if (b >= n) break;
      rb = blocks[b];
    }
  }
  cyc_blocks += clock64() - t_a;
  double2* row = reinterpret_cast<double2*>(s_red + (size_t)tid * RS);
#pragma unroll
  for (int k = 0; k < RS / 2; ++k) row[k] = make_double2(acc[2 * k], acc[2 * k + 1]);
  __syncwarp();
  double mine = 0.0;
  if (lane < RS) {
    const double* col = s_red + (size_t)(warp * 32) * RS + lane;
    double s4[4] = {0.0, 0.0, 0.0, 0.0};   // four interleaved chains, then a fixed tree
#pragma unroll
    for (int r = 0; r < 32; r += 4) {
#pragma unroll
      for (int q = 0; q < 4; ++q) s4[q] += col[(r + q) * RS];
    }
    mine = (s4[0] + s4[1]) + (s4[2] + s4[3]);
  }
  s_part[warp][lane] = mine;
  __syncthreads();
  if (warp == 0) {
    static_assert(NW == 9, "fixed summation tree below is written for 9 warps");
    const double v = ((s_part[0][lane] + s_part[1][lane]) + (s_part[2][lane] + s_part[3][lane])) +
                     ((s_part[4][lane] + s_part[5][lane]) + (s_part[6][lane] + s_part[7][lane])) + s_part[8][lane];
    double* slot = &s_in[pass & 1][crank][lane];
    for (unsigned r = 0; r < csize; ++r) *cluster.map_shared_rank(slot, r) = v;
  }
  const long long t_c = clock64();
  cluster.sync();   // release / acquire: every CTA's pushes of this pass are visible
  cyc_barrier += clock64() - t_c;
  if (warp == 0) {
    // rank order, fixed tree => identical totals in every CTA (the cluster size is 8 in every launch; ranks that do
    // not exist would read zeros written at kernel start)
    const double (*in)[32] = s_in[pass & 1];
    s_tot[lane] = ((in[0][lane] + in[1][lane]) + (in[2][lane] + in[3][lane])) + ((in[4][lane] + in[5][lane]) + (in[6][lane] + in[7][lane]));
    __syncwarp();
  }
  ++pass;
}

__device__ __forceinline__ BlockRec load_first_block(const BlockRec* __restrict__ blocks, int n, unsigned crank) {
  BlockRec rb;
  rb.type = -1;
  const int gtid = first_block_index(crank, 8);
  if (gtid < n) rb = blocks[gtid];
  return rb;
}

}  // namespace

__global__ void k_pack_blocks(const double* __restrict__ packed, int n, BlockRec* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* p = packed + (size_t)i * 11;
  BlockRec r;
  r.type = (int)p[0];
  for (int k = 0; k < 3; ++k) { r.cp[k] = p[1 + k]; r.a[k] = p[4 + k]; r.b[k] = p[7 + k]; }
  r.s = p[10];   // edge / plane: interpolation ratio ; plane-norm: negative_OA_dot_norm
  r.w = 0.0;
  if (r.type == 0) {  // edge: 1/|a-b| is precomputed for the evaluation passes
    const double ex = r.a[0] - r.b[0], ey = r.a[1] - r.b[1], ez = r.a[2] - r.b[2];
    r.w = 1.0 / sqrt(ex * ex + ey * ey + ez * ez);
  }
  r.pad = 0;
  out[i] = r;
}

// all-reduce of the cluster totals over the ranks through peer memory (see PeerX in kernels.h).  Called by every thread of the
// cluster after cluster_evaluate; on return `tot` holds the sum over all ranks, bit-identical on every rank (rank-order sum).
// Low-latency protocol: every 8-byte word carries 4 bytes of payload and the 4-byte tag of the evaluation (8-byte stores are
// atomic over NVLink), so the receiver polls the data words themselves -- no memory fence and no separate flag: one one-way
// NVLink latency per exchange.  Mailboxes are double-buffered by the parity of the tag: a rank can run at most one evaluation
// ahead of a peer (it needs the peer's contribution to finish the next one).
template <typename Cluster>
__device__ __forceinline__ void peer_allreduce(Cluster& cluster, const PeerX& px, unsigned long long seq, double* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int par = (int)(seq & 1ull);
  const unsigned long long tag = (seq & 0xffffffffull) << 32;
  if (cluster.block_rank() == 0 && warp == 0) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(tot[lane]);
    const unsigned long long w0 = (bits & 0xffffffffull) | tag, w1 = (bits >> 32) | tag;
    const size_t slot = ((size_t)(par * px.world + px.rank) * 32 + lane) * 2;
    for (int r = 0; r < px.world; ++r) {   // peer stores (NVLink); my own mailbox too, so that the sum below is uniform
      volatile unsigned long long* dst = reinterpret_cast<volatile unsigned long long*>(px.box[r]) + slot;
      dst[0] = w0; dst[1] = w1;
    }
    double sum = 0.0;
    const long long t0 = clock64();
    for (int r = 0; r < px.world; ++r) {
      const volatile unsigned long long* src = reinterpret_cast<const volatile unsigned long long*>(px.box[px.rank]) + ((size_t)(par * px.world + r) * 32 + lane) * 2;
      unsigned long long a, b;
      for (;;) {
        a = src[0]; b = src[1];
        if ((a >> 32) == (tag >> 32) && (b >> 32) == (tag >> 32)) break;
        if (clock64() - t0 > 4000000000ll) { *px.err = 1; a = b = 0; break; }   // ~2 s: a peer is gone; never hang the GPU
      }
      sum += __longlong_as_double((long long)((a & 0xffffffffull) | (b << 32)));
    }
    px.gtot[par * 32 + lane] = sum;
    __threadfence();
  }
  cluster.sync();
  if (warp == 0) { tot[lane] = *reinterpret_cast<const volatile double*>(px.gtot + par * 32 + lane); __syncwarp(); }
}

template <bool GENERAL>
__device__ __forceinline__ void lm_solve_body(const Batch<LmArgs>& B, const LmParams& prm, int mode, int integrate, const PeerX& px) {
  // one cluster (8 CTAs along x) per trajectory of the batch: blockIdx.y selects it
  const LmArgs& A = B.a[blockIdx.y];
  const BlockRec* __restrict__ blocks = A.blocks;
  const int* __restrict__ n_blocks_ptr = A.n_blocks_ptr;
  const int n_blocks_host = A.n_blocks_host;
  double* __restrict__ x7 = A.x7;
  LmSummary* __restrict__ summary = A.summary;
  double* __restrict__ out28 = A.out28;
  double* __restrict__ world7 = A.world7;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) double s_red[];   // [NT][RS] transpose scratch
  __shared__ double s_part[NW][32];
  __shared__ double s_in[2][8][32];   // partial totals pushed by the 8 CTAs of the cluster, double-buffered by pass parity
  __shared__ double s_tot[2][32];   // totals of the accepted point (T.acc_buf) and of the candidate being evaluated
  __shared__ double s_x[7];
  __shared__ TrState T;
  __shared__ double s_trace[ALOAM_LM_MAX_TRACE][8];   // trace rows of this solve, flushed by tr_finish
  const int tid = threadIdx.x;
  pdl_launch_dependents();
  // Every CTA of the cluster must have started before its shared memory is written remotely (the first push happens
  // before the first barrier of a pass).  Placed before pdl_wait(): when the kernel was launched with a programmatic
  // dependency this barrier runs while the predecessor is still finishing.  (compute-sanitizer racecheck flags the
  // kernel without it: "block that might not have entered yet".)
  cluster.sync();
  pdl_wait();   // blocks / x7 are produced by the preceding kernel of the stream
  const int n = n_blocks_ptr ? *n_blocks_ptr : n_blocks_host;
  const bool writer = cluster.block_rank() == 0 && tid == 0;
  int pass = 0;
  const long long clk0 = clock64();
  const BlockRec rb0 = load_first_block(blocks, n, cluster.block_rank());

  if (tid < 7) s_x[tid] = x7[tid];
  __syncthreads();
  // one evaluation site (the evaluation body is large; duplicating it costs instruction-cache misses)
  bool first = true;
  long long cyc_eval = 0, cyc_tr = 0, cyc_blocks = 0, cyc_barrier = 0;
  const unsigned long long seq0 = (GENERAL && px.world >= 1) ? *px.seq : 0ull;
  do {
    const long long c0 = clock64();
    double* tot = s_tot[first ? 0 : 1 - T.acc_buf];
    cluster_evaluate<GENERAL>(cluster, blocks, n, rb0, first ? s_x : T.xc, prm.huber_a, s_red, s_part, s_in, tot, pass, cyc_blocks, cyc_barrier);
    if (GENERAL && px.world >= 1) peer_allreduce(cluster, px, seq0 + (unsigned long long)pass, tot);   // pass was advanced: tags start at seq0 + 1
    const long long c1 = clock64();
    cyc_eval += c1 - c0;
    if (first && mode == 1) {
      if (cluster.block_rank() == 0 && tid < 28) out28[tid] = tot[tid];
      return;   // all remote stores into this CTA preceded the cluster barrier inside cluster_evaluate
    }
    // thread 0 of EVERY CTA takes the same decision from the same totals (no broadcast needed).  The step works on a LOCAL copy
    // of the state (registers) and of nothing else in shared memory but the two totals vectors: with every field access going to
    // shared memory behind possibly-aliasing stores the step took a large share of the solve.
    // k_lm_tr_shard takes the same step.  It stays written out in both kernels: as one routine shared with k_lm_tr_shard it
    // changes k_lm_solve's register allocation and code, and k_lm_solve is on the odometry chain.
    if (tid == 0) {
      TrState t;
      int next = 0;   // 0: nothing to produce, 1: next candidate from the accepted totals, 2: from the totals just evaluated
      if (first) next = tr_start(t, s_x, tot, prm, summary, writer, s_trace, true) ? 2 : 0;
      else {
        tr_copy(t, T);
        next = tr_after_eval(t, tot, prm, s_trace, true);
        if (next == 2) t.acc_buf ^= 1;
      }
      if (next) tr_next_candidate(t, next == 2 ? tot : s_tot[t.acc_buf], prm, s_trace, true);
      tr_copy(T, t);
    }
    first = false;
    __syncthreads();
    cyc_tr += clock64() - c1;
  } while (T.go);
  if (writer) {
    if (GENERAL && px.world >= 1) *px.seq = seq0 + (unsigned long long)pass;
    tr_finish(T, x7, summary, s_trace);
    summary->cyc_total = clock64() - clk0;
    summary->cyc_eval = cyc_eval;
    summary->cyc_chol = cyc_tr;
    summary->cyc_plus = cyc_blocks;    // residual blocks of this thread (the reductions are cyc_eval - cyc_plus - cyc_grad)
    summary->cyc_grad = cyc_barrier;   // cluster barriers
    if (integrate && world7) {
      // laserOdometry.cpp:504-505  t_w += q_w * t_last_curr ; q_w = q_w * q_last_curr
      const V3 u{world7[0], world7[1], world7[2]};
      const double w = world7[3];
      const V3 v{T.x[4], T.x[5], T.x[6]};
      V3 uv = crossd(u, v);
      uv.x += uv.x; uv.y += uv.y; uv.z += uv.z;
      const V3 c2 = crossd(u, uv);
      world7[4] += v.x + w * uv.x + c2.x;
      world7[5] += v.y + w * uv.y + c2.y;
      world7[6] += v.z + w * uv.z + c2.z;
      const double ax = world7[0], ay = world7[1], az = world7[2], aw = world7[3];
      const double bx = T.x[0], by = T.x[1], bz = T.x[2], bw = T.x[3];
      world7[3] = aw * bw - ax * bx - ay * by - az * bz;
      world7[0] = aw * bx + ax * bw + ay * bz - az * by;
      world7[1] = aw * by + ay * bw + az * bx - ax * bz;
      world7[2] = aw * bz + az * bw + ax * by - ay * bx;
      if (out28) {   // mode 0: `out28` doubles as the per-scan pose slot of a stream call
#pragma unroll
        for (int k = 0; k < 7; ++k) out28[k] = world7[k];
      }
    }
  }
  // no trailing cluster barrier: the only remote accesses are the pushes that precede each pass's barrier
}

// the common solve: every block has s == 1, one GPU
__global__ void __launch_bounds__(NT, 1) k_lm_solve(const __grid_constant__ Batch<LmArgs> B, LmParams prm, int mode, int integrate) {
  PeerX none; none.world = 0; none.rank = 0; none.seq = nullptr; none.gtot = nullptr; none.err = nullptr;
  lm_solve_body<false>(B, prm, mode, integrate, none);
}
// the general solve: blocks with an interpolation ratio s != 1 (DISTORTION build, blocks handed in through the C ABI) and / or the
// all-reduce of every evaluation over NVLink peer memory (sharded scan-to-map)
__global__ void __launch_bounds__(NT, 1) k_lm_solve_x(const __grid_constant__ Batch<LmArgs> B, LmParams prm, int mode, int integrate, const __grid_constant__ PeerX px) {
  lm_solve_body<true>(B, prm, mode, integrate, px);
}

size_t lm_dynamic_smem_bytes() { return (size_t)NT * RS * sizeof(double); }

// ---------------------------------------------------------------------------------------------------------------
// Sharded solve without the peer mailbox (map split over GPUs, SURVEY.md 8e): the same trust-region logic, but every evaluation is
//   k_lm_eval_shard (this rank's blocks -> local 32-vector)  ->  all-reduce (sum, 32 doubles; comm.cu)  ->  k_lm_tr_shard
// all stream-ordered, no host round trip: the schedule is fixed (1 + max_iters evaluations); once the state says
// "stop" the remaining kernels return immediately.  Every rank runs the identical step on identical totals.
size_t lm_state_bytes() { return sizeof(TrState); }

__global__ void __launch_bounds__(NT, 1) k_lm_eval_shard(const BlockRec* __restrict__ blocks, const int* __restrict__ n_ptr, int n_host,
                                                         const double* __restrict__ x7, void* state, int first, double huber_a, double* __restrict__ local32) {
  const int n = n_ptr ? *n_ptr : n_host;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) double s_red[];
  __shared__ double s_part[NW][32];
  __shared__ double s_in[2][8][32];
  __shared__ double s_tot[32];
  __shared__ double s_x[7];
  const TrState* T = reinterpret_cast<const TrState*>(state);
  const int tid = threadIdx.x;
  cluster.sync();   // all CTAs of the cluster have started before the first remote shared-memory store
  const bool active = first || T->go;   // uniform over the grid and over all ranks
  if (tid < 7) s_x[tid] = first ? x7[tid] : T->xc[tid];
  __syncthreads();
  int pass = 0;
  if (active) {
    const BlockRec rb0 = load_first_block(blocks, n, cluster.block_rank());
    long long cyc_unused0 = 0, cyc_unused1 = 0;
    cluster_evaluate<true>(cluster, blocks, n, rb0, s_x, huber_a, s_red, s_part, s_in, s_tot, pass, cyc_unused0, cyc_unused1);
    if (cluster.block_rank() == 0 && tid < 32) local32[tid] = tid < RS ? s_tot[tid] : 0.0;
  } else if (cluster.block_rank() == 0 && tid < 32) {
    local32[tid] = 0.0;
  }
}

// The step of the cluster kernel (lm_solve_body) on the state in global memory.  It ends the solve by the last evaluation of the
// schedule at the latest: every candidate costs an iteration and the max_iters-th is the last one produced.
__global__ void k_lm_tr_shard(void* state, const double* __restrict__ tot32, double* __restrict__ x7, int first, LmParams prm,
                              LmSummary* __restrict__ summary) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  TrState& T = *reinterpret_cast<TrState*>(state);
  if (!first && !T.go) return;   // the solve has ended at an earlier evaluation
  int next;   // 0: nothing to produce, 1: next candidate from the accepted totals, 2: from the totals just evaluated
  if (first) next = tr_start(T, x7, tot32, prm, summary, true, summary->trace, true) ? 2 : 0;
  else next = tr_after_eval(T, tot32, prm, summary->trace, true);
  if (next) tr_next_candidate(T, next == 2 ? tot32 : T.acc, prm, summary->trace, true);
  // the host issues the all-reduce into one fixed buffer, so the accepted point's totals are copied out of it
  if (first || next == 2) { for (int k = 0; k < 28; ++k) T.acc[k] = tot32[k]; }
  if (!T.go) tr_finish(T, x7, summary);
}

}  // namespace aloam
