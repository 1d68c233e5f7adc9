// p3p.cuh -- the minimal solver of resection with known intrinsics (absolute pose from three 2D-3D correspondences)
// and the inverse distortion that feeds it.  Device code; every translation unit that includes it is compiled with
// --fmad=false, and oracle/oracle_resection.cpp restates it statement for statement, so both give the same bits.
//
// Upstream (OpenMVG 1.4 SfM_Localizer::Localize -> ACKernelAdaptorResection_K<P3PSolver...>) solves P3P with Kneip's or
// Ke-Roumeliotis' closed form.  What reaches the result is the real solution set of a sample and the order its models
// are tried in; this file pins one evaluation of it from basic operations only (DESIGN.md sec. 2):
//   * Grunert's formulation: with s_i the depths along the unit bearings f_i, the three cosine-law equations
//     s_i^2 + s_j^2 - 2 s_i s_j cos(f_i, f_j) = |X_i - X_j|^2 become two conics in (u, v) = (s_2 / s_1, s_3 / s_1);
//     their difference is linear in u, and substituting u(v) leaves one quartic in v, whose coefficients are built by
//     polynomial products with fixed loop orders;
//   * the quartic by Ferrari's method on the largest real root of the resolvent cubic (solve_cubic_monic), three
//     Newton steps per root, roots tried in ascending order of v, equal roots once;
//   * per root with u, v > 0: the depths, two Gauss-Newton steps on the three cosine-law equations, then the rigid
//     motion between the orthonormal frames of the two triangles; models with a non-finite entry are dropped.
#pragma once
#include "acransac_device.cuh"

namespace r3d {
namespace p3p {

constexpr int kUndistortIters = 10;

// get_ud_pixel: inverse of the camera model's distortion by a fixed number of Newton steps (model: R3D_CAM_* 1..5;
// disto: k1 k2 k3 t1 t2 for the polynomial models, k1 k2 k3 k4 for the fisheye).  sfm_structure.cu also calls it for
// the Brown and fisheye observations it triangulates; that unit keeps FMA contraction, and its tests hold it to a
// tolerance rather than to the oracle's bits.
__device__ inline void undistort_pixel(int model, double f, double ppx, double ppy, const double* disto, double x, double y,
                                       double* xo, double* yo) {
  const double xd = (x - ppx) / f, yd = (y - ppy) / f;
  double xu = xd, yu = yd;
  if (model == 5) {
    const double rd = sqrt(xd * xd + yd * yd);
    if (rd > 1e-8) {
      double th = rd;
      for (int it = 0; it < kUndistortIters; ++it) {
        const double t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
        const double g = th * (1.0 + disto[0] * t2 + disto[1] * t4 + disto[2] * t6 + disto[3] * t8) - rd;
        const double dg = 1.0 + 3.0 * disto[0] * t2 + 5.0 * disto[1] * t4 + 7.0 * disto[2] * t6 + 9.0 * disto[3] * t8;
        th = th - g / dg;
      }
      const double ru = dm::cos_det(0.5 * R3D_PI - th) / dm::cos_det(th);  // tan(theta)
      const double s = ru / rd;
      xu = xd * s;
      yu = yd * s;
    }
  } else if (model >= 2) {
    const double k1 = disto[0], k2 = model >= 3 ? disto[1] : 0.0, k3 = model >= 3 ? disto[2] : 0.0;
    const double t1 = model == 4 ? disto[3] : 0.0, t2 = model == 4 ? disto[4] : 0.0;
    for (int it = 0; it < kUndistortIters; ++it) {
      const double r2 = xu * xu + yu * yu, r4 = r2 * r2, r6 = r4 * r2;
      const double c = 1.0 + k1 * r2 + k2 * r4 + k3 * r6;
      const double dc = k1 + 2.0 * k2 * r2 + 3.0 * k3 * r4;
      const double fx = xu * c + t2 * (r2 + 2.0 * xu * xu) + 2.0 * t1 * xu * yu - xd;
      const double fy = yu * c + t1 * (r2 + 2.0 * yu * yu) + 2.0 * t2 * xu * yu - yd;
      const double a00 = c + 2.0 * xu * xu * dc + 6.0 * t2 * xu + 2.0 * t1 * yu;
      const double a01 = 2.0 * xu * yu * dc + 2.0 * t2 * yu + 2.0 * t1 * xu;
      const double a11 = c + 2.0 * yu * yu * dc + 6.0 * t1 * yu + 2.0 * t2 * xu;
      const double det = a00 * a11 - a01 * a01;
      if (det == 0.0) break;
      const double dx = (a11 * fx - a01 * fy) / det, dy = (a00 * fy - a01 * fx) / det;
      xu = xu - dx;
      yu = yu - dy;
    }
  }
  *xo = f * xu + ppx;
  *yo = f * yu + ppy;
}

// real roots of y^2 + b y + c
__device__ inline int quadratic_roots(double b, double c, double* r) {
  const double disc = b * b - 4.0 * c;
  if (!(disc >= 0.0)) return 0;
  const double s = sqrt(disc);
  r[0] = (-b - s) / 2.0;
  r[1] = (-b + s) / 2.0;
  return 2;
}

// real roots of v^4 + a v^3 + b v^2 + c v + d, ascending, polished
__device__ inline int quartic_roots(double a, double b, double c, double d, double* roots) {
  const double a2 = a * a;
  const double p = b - 3.0 * a2 / 8.0;
  const double q = c - a * b / 2.0 + a2 * a / 8.0;
  const double r = d - a * c / 4.0 + a2 * b / 16.0 - 3.0 * a2 * a2 / 256.0;
  double y[4];
  int n = 0;
  double m0, m1, m2;
  const int nc = solve_cubic_monic(p, p * p / 4.0 - r, -(q * q) / 8.0, &m0, &m1, &m2);
  double m = m0;
  if (nc == 3) m = fmax(m0, fmax(m1, m2));
  if (m > 0.0 && q != 0.0) {
    const double s = sqrt(2.0 * m);
    const double h = p / 2.0 + m, k = q / (2.0 * s);
    n += quadratic_roots(s, h - k, y + n);
    n += quadratic_roots(-s, h + k, y + n);
  } else {  // q = 0: biquadratic
    double z[2];
    const int nz = quadratic_roots(p, r, z);
    for (int i = 0; i < nz; ++i)
      if (z[i] >= 0.0) {
        const double s = sqrt(z[i]);
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
  for (int i = 1; i < n; ++i)  // insertion sort (n <= 4)
    for (int j = i; j > 0 && roots[j] < roots[j - 1]; --j) {
      const double t = roots[j]; roots[j] = roots[j - 1]; roots[j - 1] = t;
    }
  return n;
}

// orthonormal frame (rows e1, e2, e3) of the triangle A B C; false when it is degenerate
__device__ inline bool triangle_frame(const double* A, const double* B, const double* C, double* E) {
  const double u[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]};
  const double w[3] = {C[0] - A[0], C[1] - A[1], C[2] - A[2]};
  const double nu = u[0] * u[0] + u[1] * u[1] + u[2] * u[2];
  const double nw = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  const double c[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
  const double ncr = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
  if (!(nu > 0.0) || !(nw > 0.0) || !(ncr > 1e-20 * (nu * nw))) return false;
  const double su = sqrt(nu), sc = sqrt(ncr);
  for (int i = 0; i < 3; ++i) {
    E[i] = u[i] / su;
    E[6 + i] = c[i] / sc;
  }
  E[3] = E[7] * E[2] - E[8] * E[1];
  E[4] = E[8] * E[0] - E[6] * E[2];
  E[5] = E[6] * E[1] - E[7] * E[0];
  return true;
}

// K = f, ppx, ppy; X: three world points (3 x 3); x: their undistorted pixels (3 x 2); P: up to four 3 x 4 row-major
// K [R | t].  Returns the number of models.
__device__ inline int solve(const double* K, const double* X, const double* x, double* P) {
  double f[9];
  for (int i = 0; i < 3; ++i) bearing(K, x[2 * i], x[2 * i + 1], f + 3 * i);
  double EX[9];
  if (!triangle_frame(X, X + 3, X + 6, EX)) return 0;
  double dd[3];  // |X2 - X3|^2, |X1 - X3|^2, |X1 - X2|^2
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
  // u^2 - 2 cg u + q1(v) = 0 and u^2 - 2 ca v u + q2(v) = 0; d = q2 - q1, e = 2 (ca v - cg), u = d / e
  const double q1[3] = {1.0 - C, 2.0 * C * cb, -C};
  const double d[3] = {C - A - 1.0, 2.0 * cb * (A - C), 1.0 - A + C};
  const double e[2] = {-2.0 * cg, 2.0 * ca};
  // g = d^2 - 2 cg d e + q1 e^2
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
    s[0] = sqrt(b2 / den);
    s[1] = u * s[0];
    s[2] = v * s[0];
    for (int it = 0; it < 2; ++it) {  // Gauss-Newton on the three cosine-law equations
      const double F0 = s[1] * s[1] + s[2] * s[2] - 2.0 * s[1] * s[2] * ca - a2;
      const double F1 = s[0] * s[0] + s[2] * s[2] - 2.0 * s[0] * s[2] * cb - b2;
      const double F2 = s[0] * s[0] + s[1] * s[1] - 2.0 * s[0] * s[1] * cg - c2;
      const double J[9] = {0.0, 2.0 * s[1] - 2.0 * s[2] * ca, 2.0 * s[2] - 2.0 * s[1] * ca,
                           2.0 * s[0] - 2.0 * s[2] * cb, 0.0, 2.0 * s[2] - 2.0 * s[0] * cb,
                           2.0 * s[0] - 2.0 * s[1] * cg, 2.0 * s[1] - 2.0 * s[0] * cg, 0.0};
      const double c00 = J[4] * J[8] - J[5] * J[7], c01 = J[5] * J[6] - J[3] * J[8], c02 = J[3] * J[7] - J[4] * J[6];
      const double det = J[0] * c00 + J[1] * c01 + J[2] * c02;
      if (det == 0.0) break;
      const double i00 = c00 / det, i01 = (J[2] * J[7] - J[1] * J[8]) / det, i02 = (J[1] * J[5] - J[2] * J[4]) / det;
      const double i10 = c01 / det, i11 = (J[0] * J[8] - J[2] * J[6]) / det, i12 = (J[2] * J[3] - J[0] * J[5]) / det;
      const double i20 = c02 / det, i21 = (J[1] * J[6] - J[0] * J[7]) / det, i22 = (J[0] * J[4] - J[1] * J[3]) / det;
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

}  // namespace p3p
}  // namespace r3d
