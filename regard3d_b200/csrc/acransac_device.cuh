// acransac_device.cuh -- device functions of the AC-RANSAC kernels (acransac_fused.cu: the persistent one-CTA-per-pair
// kernel; p3p.cuh builds on the solvers and residuals here).  Every translation unit that includes
// this header MUST be compiled with --fmad=false (regard3d_b200/build.py): each double operation rounds once, exactly
// like the host arithmetic of the CPU restatement, so discrete decisions are reproducible (see detmath.cuh).
// Upstream semantics: SURVEY.md Appendix A.4-A.6.
#pragma once
#include "acransac.cuh"
#include "detmath.cuh"
#include "fivepoint.cuh"

#include <cfloat>

namespace r3d {

// ------------------------------------------------------------------------------------------------
// numeric/poly.h SolveCubicPolynomial (closed form), evaluated with detmath
// ------------------------------------------------------------------------------------------------
__device__ inline int solve_cubic_monic(double a, double b, double c, double* x0, double* x1, double* x2) {
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
    const double sqrtQ = sqrt(Q);
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
    const double sqrtQ = sqrt(Q);
    const double sqrtQ3 = sqrtQ * sqrtQ * sqrtQ;
    const double theta = dm::acos_det(R / sqrtQ3);
    const double norm = -2 * sqrtQ;
    double r0 = norm * dm::cos_det(theta / 3) - a / 3;
    double r1 = norm * dm::cos_det((theta + 2.0 * R3D_PI) / 3) - a / 3;
    double r2 = norm * dm::cos_det((theta - 2.0 * R3D_PI) / 3) - a / 3;
    double t;
    if (r0 > r1) { t = r0; r0 = r1; r1 = t; }
    if (r1 > r2) {
      t = r1; r1 = r2; r2 = t;
      if (r0 > r1) { t = r0; r0 = r1; r1 = t; }
    }
    *x0 = r0; *x1 = r1; *x2 = r2;
    return 3;
  }
  const double sgnR = (R >= 0 ? 1 : -1);
  const double A = -sgnR * dm::cbrt_det(fabs(R) + sqrt(R2 - Q3));
  const double B = Q / A;
  *x0 = A + B - a / 3;
  return 1;
}

// 2-D nullspace of the 7x9 epipolar system by Gaussian elimination with complete pivoting +
// Gram-Schmidt (the pencil F1 + x F2 is what matters; Eigen's JacobiSVD basis is not reproducible
// across implementations anyway).
__device__ inline bool nullspace_7x9(double (*A)[9], double* f1, double* f2) {
  int colperm[9];
  for (int j = 0; j < 9; ++j) colperm[j] = j;
  for (int r = 0; r < 7; ++r) {
    int pi = r, pj = r;
    double best = fabs(A[r][r]);
    for (int i = r; i < 7; ++i)
      for (int j = r; j < 9; ++j) {
        const double v = fabs(A[i][j]);
        if (v > best) { best = v; pi = i; pj = j; }
      }
    if (!(best > 0.0)) return false;
    if (pi != r)
      for (int j = 0; j < 9; ++j) { const double t = A[r][j]; A[r][j] = A[pi][j]; A[pi][j] = t; }
    if (pj != r) {
      for (int i = 0; i < 7; ++i) { const double t = A[i][r]; A[i][r] = A[i][pj]; A[i][pj] = t; }
      const int t = colperm[r]; colperm[r] = colperm[pj]; colperm[pj] = t;
    }
    for (int i = r + 1; i < 7; ++i) {
      const double f = A[i][r] / A[r][r];
      for (int j = r + 1; j < 9; ++j) A[i][j] = A[i][j] - f * A[r][j];
      A[i][r] = 0.0;
    }
  }
  double n[2][9];
  for (int t = 0; t < 2; ++t) {
    double z[9];
    z[7] = (t == 1) ? 1.0 : 0.0;
    z[8] = (t == 0) ? 1.0 : 0.0;
    for (int r = 6; r >= 0; --r) {
      double s = 0.0;
      for (int j = r + 1; j < 9; ++j) s = s + A[r][j] * z[j];
      z[r] = -s / A[r][r];
    }
    for (int k = 0; k < 9; ++k) n[t][colperm[k]] = z[k];
  }
  double nn = 0.0;
  for (int k = 0; k < 9; ++k) nn = nn + n[0][k] * n[0][k];
  nn = sqrt(nn);
  for (int k = 0; k < 9; ++k) f1[k] = n[0][k] / nn;
  double dp = 0.0;
  for (int k = 0; k < 9; ++k) dp = dp + n[1][k] * f1[k];
  double g[9];
  for (int k = 0; k < 9; ++k) g[k] = n[1][k] - dp * f1[k];
  double gn = 0.0;
  for (int k = 0; k < 9; ++k) gn = gn + g[k] * g[k];
  gn = sqrt(gn);
  for (int k = 0; k < 9; ++k) f2[k] = g[k] / gn;
  return true;
}

// SevenPointSolver::Solve, minimal case
__device__ inline int seven_point(const double* x1, const double* x2, double* Fout) {
  double A[7][9];
  for (int i = 0; i < 7; ++i) {
    const double x1x = x1[2 * i], x1y = x1[2 * i + 1], x2x = x2[2 * i], x2y = x2[2 * i + 1];
    A[i][0] = x2x * x1x;
    A[i][1] = x2x * x1y;
    A[i][2] = x2x;
    A[i][3] = x2y * x1x;
    A[i][4] = x2y * x1y;
    A[i][5] = x2y;
    A[i][6] = x1x;
    A[i][7] = x1y;
    A[i][8] = 1.0;
  }
  double F1[9], F2[9];
  if (!nullspace_7x9(A, F1, F2)) return 0;
  const double a = F1[0], j = F2[0], b = F1[1], k = F2[1], c = F1[2], l = F2[2], d = F1[3], m = F2[3],
               e = F1[4], n = F2[4], f = F1[5], o = F2[5], g = F1[6], p = F2[6], h = F1[7], q = F2[7],
               i = F1[8], r = F2[8];
  double P[4];
  P[0] = a * e * i + b * f * g + c * d * h - a * f * h - b * d * i - c * e * g;
  P[1] = a * e * r + a * i * n + b * f * p + b * g * o + c * d * q + c * h * m + d * h * l + e * i * j +
         f * g * k - a * f * q - a * h * o - b * d * r - b * i * m - c * e * p - c * g * n - d * i * k -
         e * g * l - f * h * j;
  P[2] = a * n * r + b * o * p + c * m * q + d * l * q + e * j * r + f * k * p + g * k * o + h * l * m +
         i * j * n - a * o * q - b * m * r - c * n * p - d * k * r - e * l * p - f * j * q - g * l * n -
         h * j * o - i * k * m;
  P[3] = j * n * r + k * o * p + l * m * q - j * o * q - k * m * r - l * n * p;
  if (P[0] == 0.0) return 0;
  double roots[3];
  const int num_roots = solve_cubic_monic(P[2] / P[3], P[1] / P[3], P[0] / P[3], roots, roots + 1, roots + 2);
  for (int kk = 0; kk < num_roots; ++kk)
    for (int t = 0; t < 9; ++t) Fout[9 * kk + t] = F1[t] + roots[kk] * F2[t];
  return num_roots;
}

// FourPointSolver::Solve (minimal case): 1-D nullspace of the 8x9 DLT system
__device__ inline bool nullspace_8x9(double (*A)[9], double* h) {
  int colperm[9];
  for (int j = 0; j < 9; ++j) colperm[j] = j;
  for (int r = 0; r < 8; ++r) {
    int pi = r, pj = r;
    double best = fabs(A[r][r]);
    for (int i = r; i < 8; ++i)
      for (int j = r; j < 9; ++j) {
        const double v = fabs(A[i][j]);
        if (v > best) { best = v; pi = i; pj = j; }
      }
    if (!(best > 0.0)) return false;
    if (pi != r)
      for (int j = 0; j < 9; ++j) { const double t = A[r][j]; A[r][j] = A[pi][j]; A[pi][j] = t; }
    if (pj != r) {
      for (int i = 0; i < 8; ++i) { const double t = A[i][r]; A[i][r] = A[i][pj]; A[i][pj] = t; }
      const int t = colperm[r]; colperm[r] = colperm[pj]; colperm[pj] = t;
    }
    for (int i = r + 1; i < 8; ++i) {
      const double f = A[i][r] / A[r][r];
      for (int j = r + 1; j < 9; ++j) A[i][j] = A[i][j] - f * A[r][j];
      A[i][r] = 0.0;
    }
  }
  double z[9];
  z[8] = 1.0;
  for (int r = 7; r >= 0; --r) {
    double s = 0.0;
    for (int j = r + 1; j < 9; ++j) s = s + A[r][j] * z[j];
    z[r] = -s / A[r][r];
  }
  double nn = 0.0;
  for (int k = 0; k < 9; ++k) nn = nn + z[k] * z[k];
  nn = sqrt(nn);
  for (int k = 0; k < 9; ++k) h[colperm[k]] = z[k] / nn;
  return true;
}

__device__ inline int four_point(const double* x, const double* y, double* Hout) {
  double L[8][9];
  for (int i = 0; i < 4; ++i) {
    const double xx = x[2 * i], xy = x[2 * i + 1], yx = y[2 * i], yy = y[2 * i + 1];
    double* a = L[2 * i];
    double* b = L[2 * i + 1];
    a[0] = xx; a[1] = xy; a[2] = 1.0; a[3] = 0.0; a[4] = 0.0; a[5] = 0.0; a[6] = -yx * xx; a[7] = -yx * xy; a[8] = -yx;
    b[0] = 0.0; b[1] = 0.0; b[2] = 0.0; b[3] = xx; b[4] = xy; b[5] = 1.0; b[6] = -yy * xx; b[7] = -yy * xy; b[8] = -yy;
  }
  return nullspace_8x9(L, Hout) ? 1 : 0;
}

// bearing vector of a pixel: (K^-1 [x y 1]^T).normalized(), K = [f 0 ppx; 0 f ppy; 0 0 1]
// (openMVG Pinhole_Intrinsic::operator())
__device__ __forceinline__ void bearing(const double* K, double x, double y, double* b) {
  const double kinv00 = 1.0 / K[0], kinv02 = -K[1] / K[0], kinv12 = -K[2] / K[0];
  const double bx = kinv00 * x + kinv02, by = kinv00 * y + kinv12, bz = 1.0;
  const double n = sqrt((bx * bx + by * by) + bz * bz);
  b[0] = bx / n; b[1] = by / n; b[2] = bz / n;
}

// FundamentalFromEssential: F = K2^-T E K1^-1
__device__ inline void fundamental_from_essential(const double* E, const double* K1, const double* K2, double* F) {
  const double k1[9] = {1.0 / K1[0], 0.0, -K1[1] / K1[0], 0.0, 1.0 / K1[0], -K1[2] / K1[0], 0.0, 0.0, 1.0};
  const double k2[9] = {1.0 / K2[0], 0.0, -K2[1] / K2[0], 0.0, 1.0 / K2[0], -K2[2] / K2[0], 0.0, 0.0, 1.0};
  double T[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double a = 0.0;
      for (int k = 0; k < 3; ++k) a = a + k2[3 * k + r] * E[3 * k + c];
      T[3 * r + c] = a;
    }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double a = 0.0;
      for (int k = 0; k < 3; ++k) a = a + T[3 * r + k] * k1[3 * k + c];
      F[3 * r + c] = a;
    }
}

// SymmetricEpipolarDistanceError::Error
__device__ __forceinline__ double sym_epi_error(const double* F, double x1x, double x1y, double x2x, double x2y) {
  const double Fx0 = F[0] * x1x + F[1] * x1y + F[2];
  const double Fx1 = F[3] * x1x + F[4] * x1y + F[5];
  const double Fx2 = F[6] * x1x + F[7] * x1y + F[8];
  const double Fty0 = F[0] * x2x + F[3] * x2y + F[6];
  const double Fty1 = F[1] * x2x + F[4] * x2y + F[7];
  const double yFx = x2x * Fx0 + x2y * Fx1 + Fx2;
  return (yFx * yFx) * (1.0 / (Fx0 * Fx0 + Fx1 * Fx1) + 1.0 / (Fty0 * Fty0 + Fty1 * Fty1)) / 4.0;
}

// fundamental::kernel::EpipolarDistanceError::Error: squared distance of x2 to the epipolar line F x1 (pixels^2)
__device__ __forceinline__ double epi_dist_error(const double* F, double x1x, double x1y, double x2x, double x2y) {
  const double Fx0 = F[0] * x1x + F[1] * x1y + F[2];
  const double Fx1 = F[3] * x1x + F[4] * x1y + F[5];
  const double Fx2 = F[6] * x1x + F[7] * x1y + F[8];
  const double yFx = x2x * Fx0 + x2y * Fx1 + Fx2;
  return (yFx * yFx) / (Fx0 * Fx0 + Fx1 * Fx1);
}

// homography::kernel::AsymmetricError::Error
__device__ __forceinline__ double asym_error(const double* H, double x1x, double x1y, double x2x, double x2y) {
  const double hx = H[0] * x1x + H[1] * x1y + H[2];
  const double hy = H[3] * x1x + H[4] * x1y + H[5];
  const double hw = H[6] * x1x + H[7] * x1y + H[8];
  const double ex = x2x - hx / hw;
  const double ey = x2y - hy / hw;
  return ex * ex + ey * ey;
}

// resection::kernel::PoseResectionKernel / SquaredPixelReprojectionError: |x - (P X)_xy / (P X)_w|^2, P 3 x 4 row-major
__device__ __forceinline__ double resect_error(const double* P, double X, double Y, double Z, double x, double y) {
  const double px = P[0] * X + P[1] * Y + P[2] * Z + P[3];
  const double py = P[4] * X + P[5] * Y + P[6] * Z + P[7];
  const double pw = P[8] * X + P[9] * Y + P[10] * Z + P[11];
  const double ex = x - px / pw;
  const double ey = y - py / pw;
  return ex * ex + ey * ey;
}

__device__ __forceinline__ bool key_less(double ea, uint32_t ia, double eb, uint32_t ib) {
  return (ea < eb) || (ea == eb && ia < ib);
}

// Compact the residuals <= max_thr of model F into shared memory and sort them ascending by
// (residual, index).  Returns the count c; se/si hold the sorted keys in [0, c).
// WITH_INDEX = false (scoring): only the residual VALUES are sorted -- the NFA scan reads nothing else and
// ties are indistinguishable there -- which halves the shared-memory traffic of the bitonic network.
template <int MODEL, bool WITH_INDEX>
__device__ uint32_t residuals_sorted(const AcPair& pr, const double2* __restrict__ x1, const double2* __restrict__ x2,
                                     const double* Fm, double* se, uint32_t* si, uint32_t cap, uint32_t* s_count,
                                     const double* __restrict__ x3 = nullptr) {
  if (threadIdx.x == 0) *s_count = 0;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < pr.M; i += blockDim.x) {
    const double2 a = x1[pr.pt_ofs + i];
    const double2 b = x2[pr.pt_ofs + i];
    const double e = MODEL == 0   ? sym_epi_error(Fm, a.x, a.y, b.x, b.y)
                     : MODEL == 1 ? asym_error(Fm, a.x, a.y, b.x, b.y)
                     : MODEL == 2 ? epi_dist_error(Fm, a.x, a.y, b.x, b.y)
                                  : resect_error(Fm, a.x, a.y, x3[pr.pt_ofs + i], b.x, b.y);
    if (e <= pr.max_thr) {  // false for NaN
      const uint32_t pos = atomicAdd(s_count, 1u);
      if (pos < cap) {
        se[pos] = e;
        if (WITH_INDEX) si[pos] = i;
      }
    }
  }
  __syncthreads();
  uint32_t c = *s_count;
  if (c > cap) c = cap;
  uint32_t p2 = 1;
  while (p2 < c) p2 <<= 1;
  for (uint32_t i = c + threadIdx.x; i < p2; i += blockDim.x) {
    se[i] = DBL_MAX;
    if (WITH_INDEX) si[i] = 0xffffffffu;
  }
  __syncthreads();
  for (uint32_t size = 2; size <= p2; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = threadIdx.x; t < (p2 >> 1); t += blockDim.x) {
        const uint32_t lo = (t / stride) * (stride << 1) + (t % stride);
        const uint32_t hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const double ea = se[lo], eb = se[hi];
        if (WITH_INDEX) {
          const uint32_t ia = si[lo], ib = si[hi];
          const bool swap = up ? key_less(eb, ib, ea, ia) : key_less(ea, ia, eb, ib);
          if (swap) { se[lo] = eb; se[hi] = ea; si[lo] = ib; si[hi] = ia; }
        } else {
          const bool swap = up ? (eb < ea) : (ea < eb);
          if (swap) { se[lo] = eb; se[hi] = ea; }
        }
      }
      __syncthreads();
    }
  }
  return c;
}


// bestNFA over the sorted residuals se[0, c) (robust_estimation/robust_estimator_ACRansac.hpp): k = sizeSample+1 .. c
// (the upstream loop stops at the first residual > maxThreshold; se holds only those <= it), the FIRST minimum in
// ascending k is kept.  Block-wide; the result is valid in every thread.  s_nfa / s_k: >= blockDim.x / 32 entries.
struct NfaBest { double nfa, err; uint32_t k; };
template <int MODEL>
__device__ NfaBest nfa_scan_sorted(const AcPair& pr, const double* se, uint32_t c, const float* __restrict__ lcn,
                                   const float* __restrict__ logc_k, double* s_nfa, uint32_t* s_k) {
  constexpr uint32_t NS = ac_min_samples(MODEL);      // Kernel::MINIMUM_SAMPLES
  const double mult_error = (MODEL == 1 || MODEL == 3) ? 1.0 : 0.5;   // point-to-point : point-to-line
  double best = DBL_MAX * 2.0;  // +inf
  uint32_t best_k = NS;
  for (uint32_t k = NS + 1 + threadIdx.x; k <= c; k += blockDim.x) {
    const double logalpha = pr.logalpha0 + mult_error * dm::log10_det(se[k - 1] + (double)FLT_EPSILON);
    const double nfa = pr.loge0 + logalpha * (double)(k - NS) + (double)lcn[k] + (double)logc_k[k];
    if (nfa < best) { best = nfa; best_k = k; }  // ascending k per thread: first minimum is kept
  }
  for (int o = 16; o >= 1; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const uint32_t ok = __shfl_xor_sync(0xffffffffu, best_k, o);
    if (ob < best || (ob == best && ok < best_k)) { best = ob; best_k = ok; }
  }
  if ((threadIdx.x & 31u) == 0) { s_nfa[threadIdx.x >> 5] = best; s_k[threadIdx.x >> 5] = best_k; }
  __syncthreads();
  best = s_nfa[0];
  best_k = s_k[0];
  for (uint32_t w = 1; w < (blockDim.x >> 5); ++w)
    if (s_nfa[w] < best || (s_nfa[w] == best && s_k[w] < best_k)) { best = s_nfa[w]; best_k = s_k[w]; }
  NfaBest r;
  r.nfa = best;
  r.k = best_k;
  r.err = (best_k > NS && best_k <= c) ? se[best_k - 1] : 0.0;
  __syncthreads();  // s_nfa / s_k / se may be rewritten by the caller's next model
  return r;
}

}  // namespace r3d
