// oracle_resection.cpp -- CPU ORACLE (test infrastructure; see oracle_resection.h).
//
// Restates the resection step of the incremental SfM engines the reference drives
// (src/threads/R3DTriangulationThread.cpp:416-512; un-vendored OpenMVG 1.4 sfm_localizer.cpp, SURVEY.md A.12):
//   * SfM_Localizer::Localize: the pixels undistorted once (get_ud_pixel), ACRANSAC with
//     ACKernelAdaptorResection_K<P3PSolver, SquaredPixelReprojectionError, Mat34>: 3 samples, up to 4 models, residual
//     |x - pi(P X)|^2 in pixels with P = K [R | t], point-to-point a-contrario model log10(pi / (w h)), no
//     normalisation, error_max = infinity by default; rejected when minNFA >= 0 or #inliers <= 2.5 * 3.  The state
//     machine, the std::mt19937 stream, the sampling and the NFA tables are those of robust_estimator_ACRansac.hpp as
//     oracle_acransac.cpp restates them for F / H / E (that file's helpers are file-local, so the loop is written out
//     here for the 3 x 4 model and the 3-D first point);
//   * SfM_Localizer::RefinePose(pose only): Levenberg-Marquardt on angle-axis | t over the inliers, residuals on the
//     original pixels through the full camera model (orc_ba_jacobian_model), HuberLoss, the trust region of
//     oracle_ba.cpp (SURVEY.md A.7) on a dense 6 x 6 system.
// Deliberate, documented deviations (DESIGN.md sec. 2):
//   * P3P: Grunert's quartic solved by Ferrari's method with Newton polish, models in ascending order of the root
//     (upstream: Kneip / Ke-Roumeliotis; same real solution set up to rounding, another order);
//   * get_ud_pixel: a fixed number of Newton steps on the distortion map (upstream: bisection on the radius / a
//     fixed-point loop with a tolerance);
//   * no pinhole intrinsic: status NO_INTRINSIC (upstream falls back to a 6-point DLT).
// PARITY UNPINNED.
#include "oracle_resection.h"

#include "oracle_detmath.hpp"
#include "oracle_undistort.hpp"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <random>
#include <utility>
#include <vector>
#include <omp.h>

namespace orc {
namespace rs {


// numeric/poly.h SolveCubicPolynomial, as oracle_acransac.cpp
static int solve_cubic_monic(double a, double b, double c, double* x0, double* x1, double* x2) {
  const double q = a * a - 3 * b;
  const double r = 2 * a * a * a - 9 * a * b + 27 * c;
  const double Q = q / 9;
  const double R = r / 54;
  const double Q3 = Q * Q * Q;
  const double R2 = R * R;
  const double CR2 = 729 * r * r;
  const double CQ3 = 2916 * q * q * q;
  if (R == 0 && Q == 0) {
    *x0 = *x1 = *x2 = -a / 3;
    return 3;
  } else if (CR2 == CQ3) {
    const double sqrtQ = std::sqrt(Q);
    if (R > 0) {
      *x0 = -2 * sqrtQ - a / 3;
      *x1 = sqrtQ - a / 3;
      *x2 = sqrtQ - a / 3;
    } else {
      *x0 = -sqrtQ - a / 3;
      *x1 = -sqrtQ - a / 3;
      *x2 = 2 * sqrtQ - a / 3;
    }
    return 3;
  } else if (CR2 < CQ3) {
    const double sqrtQ = std::sqrt(Q);
    const double sqrtQ3 = sqrtQ * sqrtQ * sqrtQ;
    const double theta = det::acos(R / sqrtQ3);
    const double norm = -2 * sqrtQ;
    *x0 = norm * det::cos(theta / 3) - a / 3;
    *x1 = norm * det::cos((theta + 2.0 * det::kPi) / 3) - a / 3;
    *x2 = norm * det::cos((theta - 2.0 * det::kPi) / 3) - a / 3;
    if (*x0 > *x1) std::swap(*x0, *x1);
    if (*x1 > *x2) {
      std::swap(*x1, *x2);
      if (*x0 > *x1) std::swap(*x0, *x1);
    }
    return 3;
  }
  const double sgnR = (R >= 0 ? 1 : -1);
  const double A = -sgnR * det::cbrt(std::fabs(R) + std::sqrt(R2 - Q3));
  const double B = Q / A;
  *x0 = A + B - a / 3;
  return 1;
}

// Pinhole_Intrinsic::operator(): (K^-1 [x y 1]^T).normalized()
static void bearing(const double* K, double x, double y, double* b) {
  const double kinv00 = 1.0 / K[0], kinv02 = -K[1] / K[0], kinv12 = -K[2] / K[0];
  const double bx = kinv00 * x + kinv02, by = kinv00 * y + kinv12, bz = 1.0;
  const double n = std::sqrt((bx * bx + by * by) + bz * bz);
  b[0] = bx / n; b[1] = by / n; b[2] = bz / n;
}

static int quadratic_roots(double b, double c, double* r) {
  const double disc = b * b - 4.0 * c;
  if (!(disc >= 0.0)) return 0;
  const double s = std::sqrt(disc);
  r[0] = (-b - s) / 2.0;
  r[1] = (-b + s) / 2.0;
  return 2;
}

// real roots of v^4 + a v^3 + b v^2 + c v + d (Ferrari on the largest real root of the resolvent cubic), ascending
static int quartic_roots(double a, double b, double c, double d, double* roots) {
  const double a2 = a * a;
  const double p = b - 3.0 * a2 / 8.0;
  const double q = c - a * b / 2.0 + a2 * a / 8.0;
  const double r = d - a * c / 4.0 + a2 * b / 16.0 - 3.0 * a2 * a2 / 256.0;
  double y[4];
  int n = 0;
  double m0, m1, m2;
  const int nc = solve_cubic_monic(p, p * p / 4.0 - r, -(q * q) / 8.0, &m0, &m1, &m2);
  double m = m0;
  if (nc == 3) m = std::fmax(m0, std::fmax(m1, m2));
  if (m > 0.0 && q != 0.0) {
    const double s = std::sqrt(2.0 * m);
    const double h = p / 2.0 + m, k = q / (2.0 * s);
    n += quadratic_roots(s, h - k, y + n);
    n += quadratic_roots(-s, h + k, y + n);
  } else {
    double z[2];
    const int nz = quadratic_roots(p, r, z);
    for (int i = 0; i < nz; ++i)
      if (z[i] >= 0.0) {
        const double s = std::sqrt(z[i]);
        y[n++] = -s;
        y[n++] = s;
      }
  }
  for (int i = 0; i < n; ++i) {
    double v = y[i] - a / 4.0;
    for (int it = 0; it < 3; ++it) {
      const double g = (((v + a) * v + b) * v + c) * v + d;
      const double dg = ((4.0 * v + 3.0 * a) * v + 2.0 * b) * v + c;
      if (dg != 0.0) v = v - g / dg;
    }
    roots[i] = v;
  }
  for (int i = 1; i < n; ++i)
    for (int j = i; j > 0 && roots[j] < roots[j - 1]; --j) {
      const double t = roots[j]; roots[j] = roots[j - 1]; roots[j - 1] = t;
    }
  return n;
}

static bool triangle_frame(const double* A, const double* B, const double* C, double* E) {
  const double u[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]};
  const double w[3] = {C[0] - A[0], C[1] - A[1], C[2] - A[2]};
  const double nu = u[0] * u[0] + u[1] * u[1] + u[2] * u[2];
  const double nw = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  const double c[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
  const double ncr = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
  if (!(nu > 0.0) || !(nw > 0.0) || !(ncr > 1e-20 * (nu * nw))) return false;
  const double su = std::sqrt(nu), sc = std::sqrt(ncr);
  for (int i = 0; i < 3; ++i) {
    E[i] = u[i] / su;
    E[6 + i] = c[i] / sc;
  }
  E[3] = E[7] * E[2] - E[8] * E[1];
  E[4] = E[8] * E[0] - E[6] * E[2];
  E[5] = E[6] * E[1] - E[7] * E[0];
  return true;
}

static int p3p(const double* K, const double* X, const double* x, double* P) {
  double f[9];
  for (int i = 0; i < 3; ++i) bearing(K, x[2 * i], x[2 * i + 1], f + 3 * i);
  double EX[9];
  if (!triangle_frame(X, X + 3, X + 6, EX)) return 0;
  double dd[3];
  for (int k = 0; k < 3; ++k) {
    const double* A = X + 3 * ((k + 1) % 3);
    const double* B = X + 3 * ((k + 2) % 3);
    const double e0 = A[0] - B[0], e1 = A[1] - B[1], e2 = A[2] - B[2];
    dd[k] = e0 * e0 + e1 * e1 + e2 * e2;
  }
  const double a2 = dd[0], b2 = dd[1], c2 = dd[2];
  if (!(a2 > 0.0) || !(b2 > 0.0) || !(c2 > 0.0)) return 0;
  const double ca = f[3] * f[6] + f[4] * f[7] + f[5] * f[8];
  const double cb = f[0] * f[6] + f[1] * f[7] + f[2] * f[8];
  const double cg = f[0] * f[3] + f[1] * f[4] + f[2] * f[5];
  const double A = a2 / b2, C = c2 / b2;
  const double q1[3] = {1.0 - C, 2.0 * C * cb, -C};
  const double d[3] = {C - A - 1.0, 2.0 * cb * (A - C), 1.0 - A + C};
  const double e[2] = {-2.0 * cg, 2.0 * ca};
  double g[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) g[i + j] = g[i + j] + d[i] * d[j];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 2; ++j) g[i + j] = g[i + j] - 2.0 * cg * (d[i] * e[j]);
  const double e2[3] = {e[0] * e[0], 2.0 * (e[0] * e[1]), e[1] * e[1]};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) g[i + j] = g[i + j] + q1[i] * e2[j];
  if (g[4] == 0.0 || !(g[4] - g[4] == 0.0)) return 0;
  double roots[4];
  const int nr = quartic_roots(g[3] / g[4], g[2] / g[4], g[1] / g[4], g[0] / g[4], roots);
  int nm = 0;
  for (int k = 0; k < nr; ++k) {
    const double v = roots[k];
    if (k > 0 && v == roots[k - 1]) continue;
    if (!(v > 0.0)) continue;
    const double ev = e[0] + e[1] * v;
    if (ev == 0.0) continue;
    const double u = (d[0] + (d[1] + d[2] * v) * v) / ev;
    const double den = 1.0 + v * v - 2.0 * v * cb;
    if (!(u > 0.0) || !(den > 0.0)) continue;
    double s[3];
    s[0] = std::sqrt(b2 / den);
    s[1] = u * s[0];
    s[2] = v * s[0];
    for (int it = 0; it < 2; ++it) {
      const double F0 = s[1] * s[1] + s[2] * s[2] - 2.0 * s[1] * s[2] * ca - a2;
      const double F1 = s[0] * s[0] + s[2] * s[2] - 2.0 * s[0] * s[2] * cb - b2;
      const double F2 = s[0] * s[0] + s[1] * s[1] - 2.0 * s[0] * s[1] * cg - c2;
      const double J[9] = {0.0, 2.0 * s[1] - 2.0 * s[2] * ca, 2.0 * s[2] - 2.0 * s[1] * ca,
                           2.0 * s[0] - 2.0 * s[2] * cb, 0.0, 2.0 * s[2] - 2.0 * s[0] * cb,
                           2.0 * s[0] - 2.0 * s[1] * cg, 2.0 * s[1] - 2.0 * s[0] * cg, 0.0};
      const double c00 = J[4] * J[8] - J[5] * J[7], c01 = J[5] * J[6] - J[3] * J[8], c02 = J[3] * J[7] - J[4] * J[6];
      const double dt = J[0] * c00 + J[1] * c01 + J[2] * c02;
      if (dt == 0.0) break;
      const double i00 = c00 / dt, i01 = (J[2] * J[7] - J[1] * J[8]) / dt, i02 = (J[1] * J[5] - J[2] * J[4]) / dt;
      const double i10 = c01 / dt, i11 = (J[0] * J[8] - J[2] * J[6]) / dt, i12 = (J[2] * J[3] - J[0] * J[5]) / dt;
      const double i20 = c02 / dt, i21 = (J[1] * J[6] - J[0] * J[7]) / dt, i22 = (J[0] * J[4] - J[1] * J[3]) / dt;
      s[0] = s[0] - (i00 * F0 + i01 * F1 + i02 * F2);
      s[1] = s[1] - (i10 * F0 + i11 * F1 + i12 * F2);
      s[2] = s[2] - (i20 * F0 + i21 * F1 + i22 * F2);
    }
    if (!(s[0] > 0.0) || !(s[1] > 0.0) || !(s[2] > 0.0)) continue;
    double Y[9], EY[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Y[3 * i + j] = s[i] * f[3 * i + j];
    if (!triangle_frame(Y, Y + 3, Y + 6, EY)) continue;
    double R[9], t[3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[3 * i + j] = EY[i] * EX[j] + EY[3 + i] * EX[3 + j] + EY[6 + i] * EX[6 + j];
    for (int i = 0; i < 3; ++i) t[i] = Y[i] - (R[3 * i] * X[0] + R[3 * i + 1] * X[1] + R[3 * i + 2] * X[2]);
    double* Pm = P + 12 * nm;
    for (int j = 0; j < 3; ++j) {
      Pm[j] = K[0] * R[j] + K[1] * R[6 + j];
      Pm[4 + j] = K[0] * R[3 + j] + K[2] * R[6 + j];
      Pm[8 + j] = R[6 + j];
    }
    Pm[3] = K[0] * t[0] + K[1] * t[2];
    Pm[7] = K[0] * t[1] + K[2] * t[2];
    Pm[11] = t[2];
    bool finite = true;
    for (int i = 0; i < 12; ++i)
      if (!(Pm[i] - Pm[i] == 0.0)) finite = false;
    if (finite) ++nm;
  }
  return nm;
}

static double resect_error(const double* P, double X, double Y, double Z, double x, double y) {
  const double px = P[0] * X + P[1] * Y + P[2] * Z + P[3];
  const double py = P[4] * X + P[5] * Y + P[6] * Z + P[7];
  const double pw = P[8] * X + P[9] * Y + P[10] * Z + P[11];
  const double ex = x - px / pw;
  const double ey = y - py / pw;
  return ex * ex + ey * ey;
}

static void pose_from_projective(const double* K, const double* P, double* R, double* t) {
  for (int j = 0; j < 3; ++j) {
    R[6 + j] = P[8 + j];
    R[j] = (P[j] - K[1] * P[8 + j]) / K[0];
    R[3 + j] = (P[4 + j] - K[2] * P[8 + j]) / K[0];
  }
  t[2] = P[11];
  t[0] = (P[3] - K[1] * P[11]) / K[0];
  t[1] = (P[7] - K[2] * P[11]) / K[0];
}

// robust_estimator_ACRansac.hpp with the resection adaptor; xu: undistorted pixels.  Returns #inliers (0: no model).
static uint32_t acransac_p3p(const double* X, const double* xu, uint32_t M, uint32_t w, uint32_t h, const double* K, double precision_px,
                             uint32_t max_iter, std::vector<uint32_t>& vec_inliers, double* bestP, double* errorMax_out) {
  const uint32_t sizeSample = 3, MAX_MODELS = 4;
  vec_inliers.clear();
  const uint32_t nData = M;
  if (nData <= sizeSample) return 0;
  const double logalpha0 = det::log10(det::kPi / ((double)w * (double)h));
  const double multError = 1.0;
  const double maxThreshold = precision_px * precision_px;
  std::vector<uint32_t> vec_index(nData), vec_sample(sizeSample);
  std::iota(vec_index.begin(), vec_index.end(), 0);
  std::vector<std::pair<double, uint32_t>> sorted(nData);
  const double loge0 = det::log10((double)MAX_MODELS * (double)(nData - sizeSample));
  // makelogcombi_n / makelogcombi_k (float running sums; the partial sums of logcombi(k, n) are its entries for smaller k)
  std::vector<float> vlog10(nData + 1), logc_n(nData + 1), logc_k(nData + 1);
  for (uint32_t k = 0; k <= nData; ++k) vlog10[k] = std::log10((float)k);
  {
    float r = 0.f;
    logc_n[0] = 0.f;
    for (uint32_t i = 1; i <= nData / 2; ++i) {
      r += vlog10[nData - i + 1] - vlog10[i];
      logc_n[i] = r;
    }
    for (uint32_t k = nData / 2 + 1; k <= nData; ++k) logc_n[k] = (k >= nData) ? 0.f : logc_n[nData - k];
    for (uint32_t n = 0; n <= nData; ++n) {
      uint32_t k = sizeSample;
      logc_k[n] = 0.f;
      if (k >= n) continue;
      if (n - k < k) k = n - k;
      float s = 0.f;
      for (uint32_t i = 1; i <= k; ++i) s += vlog10[n - i + 1] - vlog10[i];
      logc_k[n] = s;
    }
  }
  double minNFA = std::numeric_limits<double>::infinity();
  double errorMax = std::numeric_limits<double>::infinity();
  uint32_t nIterReserve = max_iter / 10;
  uint32_t nIter = max_iter - nIterReserve;
  bool bACRansacMode = (maxThreshold == std::numeric_limits<double>::infinity());
  std::mt19937 random_generator(std::mt19937::default_seed);
  for (uint32_t iter = 0; iter < nIter; ++iter) {
    {  // UniformSample: a partial Fisher-Yates on the pool
      const uint32_t last_idx = (uint32_t)vec_index.size() - 1;
      for (uint32_t i = 0; i < sizeSample; ++i) {
        std::uniform_int_distribution<uint32_t> distribution(i, last_idx);
        std::swap(vec_index[i], vec_index[distribution(random_generator)]);
      }
      for (uint32_t i = 0; i < sizeSample; ++i) vec_sample[i] = vec_index[i];
    }
    double Xs[9], xs[6], models[48];
    for (uint32_t t = 0; t < sizeSample; ++t) {
      for (int c = 0; c < 3; ++c) Xs[3 * t + c] = X[3 * (size_t)vec_sample[t] + c];
      for (int c = 0; c < 2; ++c) xs[2 * t + c] = xu[2 * (size_t)vec_sample[t] + c];
    }
    const int nmodels = p3p(K, Xs, xs, models);
    bool better = false;
    for (int mi = 0; mi < nmodels; ++mi) {
      const double* Pm = models + 12 * mi;
      for (uint32_t i = 0; i < nData; ++i) {
        double e = resect_error(Pm, X[3 * (size_t)i], X[3 * (size_t)i + 1], X[3 * (size_t)i + 2], xu[2 * (size_t)i], xu[2 * (size_t)i + 1]);
        if (!(e == e)) e = std::numeric_limits<double>::infinity();  // NaN never is an inlier
        sorted[i] = {e, i};
      }
      if (!bACRansacMode) {
        uint32_t nInlier = 0;
        for (uint32_t i = 0; i < nData; ++i)
          if (sorted[i].first <= maxThreshold) ++nInlier;
        if (nInlier > 2.5 * sizeSample) bACRansacMode = true;
      }
      if (bACRansacMode) {
        std::sort(sorted.begin(), sorted.end());
        double best_nfa = std::numeric_limits<double>::infinity();
        uint32_t best_k = sizeSample;
        for (uint32_t k = sizeSample + 1; k <= nData && sorted[k - 1].first <= maxThreshold; ++k) {
          const double logalpha = logalpha0 + multError * det::log10(sorted[k - 1].first + (double)FLT_EPSILON);
          const double nfa = loge0 + logalpha * (double)(k - sizeSample) + (double)logc_n[k] + (double)logc_k[k];
          if (nfa < best_nfa) { best_nfa = nfa; best_k = k; }
        }
        if (best_nfa < minNFA) {
          better = true;
          minNFA = best_nfa;
          errorMax = sorted[best_k - 1].first;
          vec_inliers.resize(best_k);
          for (uint32_t i = 0; i < best_k; ++i) vec_inliers[i] = sorted[i].second;
          std::memcpy(bestP, Pm, 12 * sizeof(double));
        }
      }
    }
    if ((better && minNFA < 0) || (iter + 1 == nIter && nIterReserve)) {
      if (vec_inliers.empty()) {
        ++nIter;
        --nIterReserve;
      } else {
        vec_index = vec_inliers;
        if (nIterReserve) {
          nIter = iter + 1 + nIterReserve;
          nIterReserve = 0;
        }
      }
    }
  }
  if (minNFA >= 0) vec_inliers.clear();
  if (!(vec_inliers.size() > 2.5 * sizeSample)) vec_inliers.clear();  // SfM_Localizer: too few inliers
  *errorMax_out = errorMax;
  return (uint32_t)vec_inliers.size();
}

// ceres::RotationMatrixToAngleAxis / AngleAxisToRotationMatrix, as oracle_relpose.cpp
static void rotation_to_angle_axis(const double* R, double* aa) {
  double q[4];
  const double trace = R[0] + R[4] + R[8];
  if (trace >= 0.0) {
    double t = std::sqrt(trace + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (R[7] - R[5]) * t;
    q[2] = (R[2] - R[6]) * t;
    q[3] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = std::sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i + 1] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (R[3 * k + j] - R[3 * j + k]) * t;
    q[j + 1] = (R[3 * j + i] + R[3 * i + j]) * t;
    q[k + 1] = (R[3 * k + i] + R[3 * i + k]) * t;
  }
  const double s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  double k = 2.0;
  if (s2 > 0.0) {
    const double st = std::sqrt(s2), ct = q[0];
    const double two_theta = 2.0 * (ct < 0.0 ? std::atan2(-st, -ct) : std::atan2(st, ct));
    k = two_theta / st;
  }
  for (int i = 0; i < 3; ++i) aa[i] = q[i + 1] * k;
}

static void angle_axis_to_rotation(const double* aa, double* R) {
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > 2.220446049250313e-16) {
    const double th = std::sqrt(th2);
    const double wx = aa[0] / th, wy = aa[1] / th, wz = aa[2] / th;
    const double c = std::cos(th), s = std::sin(th), oc = 1.0 - c;
    R[0] = c + wx * wx * oc;      R[1] = wx * wy * oc - wz * s; R[2] = wy * s + wx * wz * oc;
    R[3] = wz * s + wx * wy * oc; R[4] = c + wy * wy * oc;      R[5] = -wx * s + wy * wz * oc;
    R[6] = -wy * s + wx * wz * oc; R[7] = wx * s + wy * wz * oc; R[8] = c + wz * wz * oc;
  } else {
    R[0] = 1.0;    R[1] = -aa[2]; R[2] = aa[1];
    R[3] = aa[2];  R[4] = 1.0;    R[5] = -aa[0];
    R[6] = -aa[1]; R[7] = aa[0];  R[8] = 1.0;
  }
}

static double huber_rho(double s, double a, double* rho1) {  // ceres::HuberLoss(a), as oracle_ba.cpp
  if (a <= 0.0) { *rho1 = 1.0; return s; }
  const double b = a * a;
  if (s > b) {
    const double rr = std::sqrt(s);
    *rho1 = std::max(std::numeric_limits<double>::min(), a / rr);
    return 2.0 * a * rr - b;
  }
  *rho1 = 1.0;
  return s;
}

struct Lm {  // the pose-only problem: dense 6 x 6 trust-region LM with oracle_ba.cpp's rules
  int model;
  const double* intr8;
  const double *X, *x;
  uint32_t N;
  double huber_a;

  double cost(const double* pose) const {
    double c = 0.0;
    for (uint32_t i = 0; i < N; ++i) {
      double r[2], J[30], rho1;
      orc_ba_jacobian_model(model, intr8, intr8 + 6, pose, X + 3 * (size_t)i, x + 2 * (size_t)i, r, J);
      c += 0.5 * huber_rho(r[0] * r[0] + r[1] * r[1], huber_a, &rho1);
    }
    return c;
  }
  // Corrector-scaled Jacobian columns (scale: Jacobi scaling, computed when first) -> H = J^T J (lower), g = J^T r
  void evaluate(const double* pose, bool first, double* scale, double* H, double* g) const {
    std::vector<double> rs(2 * (size_t)N), Js(12 * (size_t)N);
    for (uint32_t i = 0; i < N; ++i) {
      double r[2], J[30], rho1;
      orc_ba_jacobian_model(model, intr8, intr8 + 6, pose, X + 3 * (size_t)i, x + 2 * (size_t)i, r, J);
      huber_rho(r[0] * r[0] + r[1] * r[1], huber_a, &rho1);
      const double sq = std::sqrt(rho1);
      for (int a = 0; a < 2; ++a) {
        rs[2 * (size_t)i + a] = r[a] * sq;
        for (int k = 0; k < 6; ++k) Js[12 * (size_t)i + 6 * a + k] = J[15 * a + 6 + k] * sq;
      }
    }
    if (first)
      for (int k = 0; k < 6; ++k) {
        double n2 = 0.0;
        for (uint32_t i = 0; i < N; ++i) {
          const double j0 = Js[12 * (size_t)i + k], j1 = Js[12 * (size_t)i + 6 + k];
          n2 += j0 * j0 + j1 * j1;
        }
        scale[k] = 1.0 / (1.0 + std::sqrt(n2));
      }
    for (int i = 0; i < 36; ++i) H[i] = 0.0;
    for (int k = 0; k < 6; ++k) g[k] = 0.0;
    for (uint32_t i = 0; i < N; ++i) {
      double j0[6], j1[6];
      for (int k = 0; k < 6; ++k) {
        j0[k] = Js[12 * (size_t)i + k] * scale[k];
        j1[k] = Js[12 * (size_t)i + 6 + k] * scale[k];
      }
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b <= a; ++b) H[6 * a + b] += j0[a] * j0[b] + j1[a] * j1[b];
      for (int k = 0; k < 6; ++k) g[k] += j0[k] * rs[2 * (size_t)i] + j1[k] * rs[2 * (size_t)i + 1];
    }
  }
};

static int refine(const Lm& P, const orc_ba_options* o, double* pose, orc_ba_summary* s) {
  std::memset(s, 0, sizeof(*s));
  double scale[6], H[36], g[6];
  double cost = P.cost(pose);
  s->initial_cost = cost;
  double radius = o->initial_radius, decrease_factor = 2.0;
  P.evaluate(pose, true, scale, H, g);
  auto grad_max = [&]() {
    double m = 0.0;
    for (int j = 0; j < 6; ++j) m = std::max(m, std::fabs(g[j] / scale[j]));
    return m;
  };
  int termination = 0;
  if (grad_max() <= o->gradient_tolerance) termination = 2;
  else
    for (uint32_t iter = 1; iter <= o->max_iterations; ++iter) {
      s->iterations = iter;
      double D2[6], A[36], b[6], delta[6];
      for (int j = 0; j < 6; ++j) D2[j] = std::min(std::max(H[7 * j], 1e-6), 1e32) / radius;
      for (int i = 0; i < 6; ++i) {
        for (int j = 0; j <= i; ++j) A[6 * i + j] = H[6 * i + j] + (i == j ? D2[i] : 0.0);
        b[i] = -g[i];
      }
      bool pd = true;
      for (int j = 0; j < 6 && pd; ++j) {
        double d = A[6 * j + j];
        for (int t = 0; t < j; ++t) d -= A[6 * j + t] * A[6 * j + t];
        if (!(d > 0.0)) { pd = false; break; }
        d = std::sqrt(d);
        A[6 * j + j] = d;
        for (int i = j + 1; i < 6; ++i) {
          double v = A[6 * i + j];
          for (int t = 0; t < j; ++t) v -= A[6 * i + t] * A[6 * j + t];
          A[6 * i + j] = v / d;
        }
      }
      bool step_ok = pd;
      double model_cost_change = 0.0;
      if (pd) {
        for (int i = 0; i < 6; ++i) {
          double v = b[i];
          for (int t = 0; t < i; ++t) v -= A[6 * i + t] * b[t];
          b[i] = v / A[6 * i + i];
        }
        for (int i = 5; i >= 0; --i) {
          double v = b[i];
          for (int t = i + 1; t < 6; ++t) v -= A[6 * t + i] * b[t];
          b[i] = v / A[6 * i + i];
        }
        double m = 0.0;
        for (int j = 0; j < 6; ++j) {
          delta[j] = b[j];
          m += delta[j] * (D2[j] * delta[j] - g[j]);
        }
        model_cost_change = 0.5 * m;
        step_ok = model_cost_change > 0.0;
      }
      bool accepted = false;
      if (step_ok) {
        double dn = 0.0, xn = 0.0, pose_new[6];
        for (int j = 0; j < 6; ++j) {
          const double d = delta[j] * scale[j];
          dn += d * d;
          xn += pose[j] * pose[j];
          pose_new[j] = pose[j] + d;
        }
        if (std::sqrt(dn) <= o->parameter_tolerance * (std::sqrt(xn) + o->parameter_tolerance)) {
          termination = 3;
          break;
        }
        const double new_cost = P.cost(pose_new);
        const double relative_decrease = (cost - new_cost) / model_cost_change;
        if (relative_decrease > 1e-3) {
          accepted = true;
          std::memcpy(pose, pose_new, sizeof(pose_new));
          const double cost_change = cost - new_cost;
          const double t = 2.0 * relative_decrease - 1.0;
          radius = radius / std::max(1.0 / 3.0, 1.0 - t * t * t);
          radius = std::min(1e16, radius);
          decrease_factor = 2.0;
          ++s->successful_steps;
          const bool ftol = std::fabs(cost_change) < o->function_tolerance * cost;
          cost = new_cost;
          P.evaluate(pose, false, scale, H, g);
          if (ftol) { termination = 1; break; }
          if (grad_max() <= o->gradient_tolerance) { termination = 2; break; }
        }
      }
      if (!accepted) {
        radius = radius / decrease_factor;
        decrease_factor *= 2.0;
        if (radius < 1e-32) { termination = 4; break; }
      }
    }
  s->termination = termination;
  s->final_cost = cost;
  return termination;
}

static void set_pose(orc_resection_result* r, const double* R, const double* t) {
  std::memcpy(r->rotation, R, 9 * sizeof(double));
  std::memcpy(r->translation, t, 3 * sizeof(double));
  for (int i = 0; i < 3; ++i) r->center[i] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
}

}  // namespace rs
}  // namespace orc

using namespace orc::rs;

extern "C" {

int orc_p3p(const double* K, const double* X, const double* x, double* P) { return p3p(K, X, x, P); }

void orc_undistort(int model, const double* intr8, const double* xy, uint32_t n, double* out) {
  for (uint32_t i = 0; i < n; ++i)
    orc::undistort_newton(model, intr8[0], intr8[1], intr8[2], intr8 + 3, xy[2 * (size_t)i], xy[2 * (size_t)i + 1],
                          out + 2 * (size_t)i, out + 2 * (size_t)i + 1);
}

int orc_resect_refine(int model, const double* intr8, const double* X, const double* x, uint32_t N, const orc_ba_options* o,
                      double* pose, orc_ba_summary* s) {
  const Lm P{model, intr8, X, x, N, o->huber_a};
  return refine(P, o, pose, s);
}

int orc_resect_view(const double* X, const double* x, uint32_t M, uint32_t width, uint32_t height, int model,
                    const double* intr8, const orc_resection_options* o, orc_resection_result* r, uint32_t* inliers) {
  const uint32_t id = r->view_id;
  std::memset(r, 0, sizeof(*r));
  r->view_id = id;
  r->lm_termination = -1;
  if (M <= 3) return r->status = ORC_RESECT_TOO_FEW;
  if (!(intr8[0] > 0.0)) return r->status = ORC_RESECT_NO_INTRINSIC;
  std::vector<double> xu(2 * (size_t)M);
  orc_undistort(model, intr8, x, M, xu.data());
  std::vector<uint32_t> inl;
  double P[12], errorMax;
  const uint32_t n = acransac_p3p(X, xu.data(), M, width, height, intr8, o->precision_px, o->max_iter, inl, P, &errorMax);
  if (n == 0) return r->status = ORC_RESECT_NO_MODEL;
  r->status = ORC_RESECT_OK;
  r->n_inliers = n;
  r->found_residual_precision = std::sqrt(errorMax);
  std::memcpy(inliers, inl.data(), inl.size() * sizeof(uint32_t));
  pose_from_projective(intr8, P, r->rotation_ransac, r->translation_ransac);
  set_pose(r, r->rotation_ransac, r->translation_ransac);
  if (!o->refine) return r->status;
  std::vector<double> Xi(3 * (size_t)n), xi(2 * (size_t)n);
  for (uint32_t k = 0; k < n; ++k) {
    for (int c = 0; c < 3; ++c) Xi[3 * (size_t)k + c] = X[3 * (size_t)inl[k] + c];
    for (int c = 0; c < 2; ++c) xi[2 * (size_t)k + c] = x[2 * (size_t)inl[k] + c];
  }
  double pose[6];
  rotation_to_angle_axis(r->rotation_ransac, pose);
  for (int i = 0; i < 3; ++i) pose[3 + i] = r->translation_ransac[i];
  orc_ba_summary s;
  orc_resect_refine(model, intr8, Xi.data(), xi.data(), n, &o->ba, pose, &s);
  r->lm_iterations = s.iterations;
  r->lm_successful_steps = s.successful_steps;
  r->lm_termination = s.termination;
  r->lm_initial_cost = s.initial_cost;
  r->lm_final_cost = s.final_cost;
  if (s.termination == 4) return r->status;  // the solve failed: the AC-RANSAC pose stays
  double R[9];
  angle_axis_to_rotation(pose, R);
  set_pose(r, R, pose + 3);
  return r->status;
}

void orc_resect_views(uint32_t n, const uint64_t* first, const uint64_t* count, const uint32_t* widths, const uint32_t* heights,
                      const int* models, const double* intr8, const double* X, const double* x, const orc_resection_options* o,
                      orc_resection_result* out, uint32_t* inl, uint64_t* inl_ofs, int n_threads) {
  if (n_threads <= 0) n_threads = omp_get_max_threads();
  std::vector<std::vector<uint32_t>> res(n);
#pragma omp parallel for schedule(dynamic) num_threads(n_threads)
  for (int64_t v = 0; v < (int64_t)n; ++v) {
    res[v].resize(std::max<uint64_t>(count[v], 1));
    orc_resect_view(X + 3 * first[v], x + 2 * first[v], (uint32_t)count[v], widths[v], heights[v], models[v], intr8 + 8 * (size_t)v, o,
                    &out[v], res[v].data());
    res[v].resize(out[v].n_inliers);
  }
  uint64_t ofs = 0;
  for (uint32_t v = 0; v < n; ++v) {
    inl_ofs[v] = ofs;
    std::memcpy(inl + ofs, res[v].data(), res[v].size() * sizeof(uint32_t));
    ofs += res[v].size();
  }
  inl_ofs[n] = ofs;
}

}  // extern "C"
