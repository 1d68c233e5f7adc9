// lm_trust_region.cuh -- the trust-region policy of Ceres' Levenberg-Marquardt, shared by the library's least-squares
// solvers: bundle adjustment (ba.cu) and rotation and translation averaging (averaging.cuh's averaging_lm, for
// rotavg.cu and transavg.cu) drive it from the host, the two-view bundle adjustment (relpose.cu, k_relpose_ba) and the
// pose refinement (resection.cu, k_resect_refine) from every thread of a CTA.  Policy only: it launches nothing, synchronises nothing and reads no
// memory; the callers keep their evaluations, linear solves and data movement.  The CPU restatements under oracle/ keep
// their own copies of these rules on purpose: they are the independent references the solvers are tested against.
//
// Basic IEEE operations only (plus sqrt, fmin, fmax).  The device side may only be used from the translation units that
// build.py compiles with --fmad=false (NO_FMAD): there it computes what the host side computes, bit for bit.  ba.cu is
// compiled with --fmad=true and uses the host side only.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/r3dgpu.h"
#include "relpose_math.cuh"  // R3D_RP_HD

namespace r3d {

struct LmParams {
  uint32_t max_iterations;
  double huber_a, function_tolerance, gradient_tolerance, parameter_tolerance, initial_radius;
};

inline LmParams lm_params(const r3d_ba_options& o) {
  LmParams p;
  p.max_iterations = o.max_iterations;
  p.huber_a = o.huber_a;
  p.function_tolerance = o.function_tolerance;
  p.gradient_tolerance = o.gradient_tolerance;
  p.parameter_tolerance = o.parameter_tolerance;
  p.initial_radius = o.initial_radius;
  return p;
}

// Every caller runs the same loop around its own solve, trial point and evaluation:
//
//   if (!lm.start(gmax))
//     for (iter = 1; iter <= lm.p.max_iterations; ++iter) {
//       lm.iterations = iter;
//       ... solve (J^T J + D^2 / lm.radius) delta = -g -> pd, model cost change mcc ...
//       bool accepted = false;
//       if (lm.step_usable(pd, mcc)) {
//         ... trial point, |step|^2, |x|^2 ...
//         if (lm.step_too_small(dn2, xn2)) break;
//         ... new_cost ...
//         if ((accepted = lm.accept(cost, new_cost, mcc))) { take the trial point; evaluate; if (lm.converged(gmax)) break; }
//       }
//       if (!accepted && lm.reject()) break;
//     }
//
// Each stop sets termination: 1 function tolerance, 2 gradient tolerance, 3 parameter tolerance, 4 trust region
// collapsed (radius below 1e-32); 0 while running and after max_iterations.
struct LmTrustRegion {
  LmParams p;
  double radius, decrease_factor;
  uint32_t iterations, successful;
  int termination;
  bool function_converged;  // the last accepted step passed the function tolerance

  R3D_RP_HD explicit LmTrustRegion(const LmParams& prm)
      : p(prm), radius(prm.initial_radius), decrease_factor(2.0), iterations(0), successful(0), termination(0),
        function_converged(false) {}

  // the gradient test at the start point (gmax = max |unscaled gradient|); true: stop before the first step
  R3D_RP_HD bool start(double gmax) {
    if (gmax <= p.gradient_tolerance) termination = 2;
    return termination != 0;
  }
  // the factorisation succeeded (pd) and the model predicts a finite decrease
  R3D_RP_HD bool step_usable(bool pd, double mcc) const { return pd && mcc > 0.0 && isfinite(mcc); }
  // |step| <= ptol (|x| + ptol), from dn2 = |step|^2 and xn2 = |x|^2 (unscaled)
  R3D_RP_HD bool step_too_small(double dn2, double xn2) {
    if (sqrt(dn2) <= p.parameter_tolerance * (sqrt(xn2) + p.parameter_tolerance)) termination = 3;
    return termination != 0;
  }
  // accepted when the relative decrease (cost - new_cost) / mcc is above 1e-3 (false for NaN): the radius grows by
  // 1 / max(1/3, 1 - (2 rho - 1)^3), capped at 1e16, and the function tolerance is tested against the old cost
  R3D_RP_HD bool accept(double cost, double new_cost, double mcc) {
    const double relative_decrease = (cost - new_cost) / mcc;
    if (!(relative_decrease > 1e-3)) return false;
    const double t = 2.0 * relative_decrease - 1.0;
    radius = radius / fmax(1.0 / 3.0, 1.0 - t * t * t);
    radius = fmin(1e16, radius);
    decrease_factor = 2.0;
    ++successful;
    function_converged = fabs(cost - new_cost) < p.function_tolerance * cost;
    return true;
  }
  // after the accepted step is evaluated (gmax at the new point): the function tolerance first, then the gradient
  R3D_RP_HD bool converged(double gmax) {
    if (function_converged) termination = 1;
    else if (gmax <= p.gradient_tolerance) termination = 2;
    return termination != 0;
  }
  // a rejected or unusable step: the radius shrinks by a factor that doubles with each consecutive rejection
  R3D_RP_HD bool reject() {
    radius = radius / decrease_factor;
    decrease_factor *= 2.0;
    if (radius < 1e-32) termination = 4;
    return termination != 0;
  }
};

// A x = b for a symmetric positive definite N x N A (row-major, lower triangle read): A's lower triangle becomes the
// Cholesky factor L and b the solution.  false (b untouched) when a pivot is not positive.
template <int N>
R3D_RP_HD bool chol_solve_small(double* A, double* b) {
  for (int j = 0; j < N; ++j) {
    double d = A[N * j + j];
    for (int t = 0; t < j; ++t) d -= A[N * j + t] * A[N * j + t];
    if (!(d > 0.0)) return false;
    d = sqrt(d);
    A[N * j + j] = d;
    for (int i = j + 1; i < N; ++i) {
      double s = A[N * i + j];
      for (int t = 0; t < j; ++t) s -= A[N * i + t] * A[N * j + t];
      A[N * i + j] = s / d;
    }
  }
  for (int i = 0; i < N; ++i) {
    double s = b[i];
    for (int t = 0; t < i; ++t) s -= A[N * i + t] * b[t];
    b[i] = s / A[N * i + i];
  }
  for (int i = N - 1; i >= 0; --i) {
    double s = b[i];
    for (int t = i + 1; t < N; ++t) s -= A[N * t + i] * b[t];
    b[i] = s / A[N * i + i];
  }
  return true;
}

#ifdef __CUDACC__
// fixed-order block reductions over kThreads threads (every thread gets the result; red: kThreads / 32 doubles)
template <int kThreads>
__device__ double block_sum_fixed(double v, double* red) {
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}
template <int kThreads>
__device__ double block_max_fixed(double v, double* red) {
  for (int o = 16; o >= 1; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kThreads / 32; ++w) s = fmax(s, red[w]);
  return s;
}
#endif

}  // namespace r3d
