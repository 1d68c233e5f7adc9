// transavg_l1.cu -- global camera translations by the L-infinity translation registration of Moulon et al. (ICCV 2013),
// Regard3D's default TRANSLATION_AVERAGING_L1 (r3d_translation_averaging_l1).
// COMPILED WITH --fmad=false (regard3d_b200/build.py), like transavg.cu: every product and sum is written out in one
// fixed order, so repeated calls are bit-identical.
//
// The linear program, on the kept edges of transavg.cu's select_edges (one relative-motion group per edge):
//   min gamma  s.t.  -gamma <= (T_J - R_IJ T_I - lambda_e u_IJ)_k <= gamma (k = 0..2),  lambda_e >= 1,  T_0 = 0,
// written as min c^T y s.t. G y + s = h, s >= 0, y = (T of the m - 1 free views, lambda per edge, gamma); per edge 7
// rows: (r_k - gamma <= 0) for k = 0..2, (-r_k - gamma <= 0) for k = 0..2, (-lambda <= -1).  Mehrotra predictor-
// corrector from T = 0, lambda = 2, gamma = 3 (strictly feasible: |u| = 1), z = 1.  Per iteration:
//   k_tl_rows    one thread per edge: residuals, D = Z / S, and the 1 x 1 Schur complement of lambda_e
//   k_tl_system  one owner CTA per free view, its incident edges in neighbour order: its 3 x 3 blocks of
//                G^T D G with lambda eliminated, its entries of the gamma row, its right-hand side rows (no atomics);
//                the gamma-gamma entry and the gamma right-hand side are per-edge partials summed by k_avg_sum
//   k_tl_norms   the residual norms, s^T z and the dual objective (fixed-order block reductions)
//   k_tl_jacobi  the reduced system of N = 3 (m - 1) + 1 scaled to a unit diagonal, and an unregularised copy of it
//   dense_cholesky (ba.cu) factors it and solves the predictor; the corrector reuses the factor through trsm3
//   (rotavg.cu); every solve gets one step of iterative refinement against the copy (k_tl_resid, trsm3, k_tl_vec)
//   k_tl_back    per edge: d lambda, ds and dz, and the ratio test per edge; k_tl_ratio the step lengths (and the
//                predictor's complementarity); k_tl_update the step.
#include "r3d_internal.cuh"
#include "averaging.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace r3d {
namespace tl {

constexpr int kRows = 7;        // LP rows per edge
constexpr int kEW = 32;         // per-edge stash of k_tl_rows (layout below)
constexpr int kNrm = 6;         // per-edge norm partials
constexpr int kRThreads = 1024;  // the one-CTA reductions
constexpr double kEta = 0.99;   // fraction of the step to the boundary
// a failed factorisation (not positive definite) is retried with kRegRel * kRegGrowth^k of the largest diagonal entry
// added to the diagonal, k = 0 .. kRegTries - 1.  Only then: a regularisation on every factorisation stalls the method.
constexpr double kRegRel = 1e-18;
constexpr double kRegGrowth = 100.0;
constexpr int kRegTries = 5;

// stash layout: p (3) = d+ + d-, q (3) = d+ - d-, zeta (3) = v+ - v-, w_I (3), w_J (3), w_gamma, V, rhs_lambda, rp (7),
// wt (7); v = z + wt is the right-hand side's multiplier, wt = (z rp - rc) / s
enum { kP = 0, kQ = 3, kZeta = 6, kWI = 9, kWJ = 12, kWG = 15, kV = 16, kRL = 17, kRp = 18, kWt = 25 };

__device__ __forceinline__ double tcoord(const double* y, uint32_t v, int k) { return v == 0 ? 0.0 : y[3 * (size_t)(v - 1) + k]; }

// r = T_J - R T_I - lambda u
__device__ __forceinline__ void edge_residual(const double* R, const double* u, const double* TI, const double* TJ, double lam,
                                              double* r) {
  for (int k = 0; k < 3; ++k) r[k] = (TJ[k] - ((R[3 * k] * TI[0] + R[3 * k + 1] * TI[1]) + R[3 * k + 2] * TI[2])) - lam * u[k];
}

// Per edge.  mode 0 (predictor): rc = s z; mode 1 (corrector): rc = s z + ds dz - sigma_mu with the predictor's ds, dz.
// Writes the stash, the partials of the gamma-gamma entry (gg) and the gamma right-hand side (gr; edge 0 also carries
// -c_gamma = -1), and in mode 0 the norm partials: max |rp|, max(0, max (G y - h)), |dual residual of lambda|,
// sum of z over the 6 gamma rows, s^T z, z_lambda.
__global__ void k_tl_rows(int mode, const uint2* __restrict__ ab, const double* __restrict__ Rij, const double* __restrict__ uij,
                          const double* __restrict__ y, const double* __restrict__ lam, const double* __restrict__ s,
                          const double* __restrict__ z, const double* __restrict__ ds, const double* __restrict__ dz, double sigma_mu,
                          uint32_t ne, uint32_t N, double* __restrict__ ew, double* __restrict__ gg, double* __restrict__ gr,
                          double* __restrict__ nrm) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  const double* R = Rij + 9 * (size_t)e;
  const double* u = uij + 3 * (size_t)e;
  double TI[3], TJ[3], r[3];
  for (int k = 0; k < 3; ++k) {
    TI[k] = tcoord(y, v.x, k);
    TJ[k] = tcoord(y, v.y, k);
  }
  const double gam = y[N - 1], la = lam[e];
  edge_residual(R, u, TI, TJ, la, r);
  double gy[kRows];  // G y - h
  for (int k = 0; k < 3; ++k) {
    gy[k] = r[k] - gam;
    gy[3 + k] = -r[k] - gam;
  }
  gy[6] = -la + 1.0;
  double* W = ew + kEW * (size_t)e;
  double d[kRows], vv[kRows];
  double pmax = 0.0, viol = 0.0, sz = 0.0, zg = 0.0;
  for (int i = 0; i < kRows; ++i) {
    const double si = s[kRows * (size_t)e + i], zi = z[kRows * (size_t)e + i];
    const double rp = gy[i] + si;
    double rc = si * zi;
    if (mode == 1) rc = (rc + ds[kRows * (size_t)e + i] * dz[kRows * (size_t)e + i]) - sigma_mu;
    const double wt = (zi * rp - rc) / si;
    d[i] = zi / si;
    vv[i] = zi + wt;
    W[kRp + i] = rp;
    W[kWt + i] = wt;
    pmax = fmax(pmax, fabs(rp));
    viol = fmax(viol, gy[i]);
    sz += si * zi;
    if (i < 6) zg += zi;
  }
  double pu[3], zeta[3];
  for (int k = 0; k < 3; ++k) {
    W[kP + k] = d[k] + d[3 + k];
    W[kQ + k] = d[k] - d[3 + k];
    pu[k] = W[kP + k] * u[k];
    zeta[k] = vv[k] - vv[3 + k];
    W[kZeta + k] = zeta[k];
  }
  for (int c = 0; c < 3; ++c) {
    W[kWI + c] = (R[c] * pu[0] + R[3 + c] * pu[1]) + R[6 + c] * pu[2];
    W[kWJ + c] = -pu[c];
  }
  const double wg = (W[kQ] * u[0] + W[kQ + 1] * u[1]) + W[kQ + 2] * u[2];
  const double V = ((pu[0] * u[0] + pu[1] * u[1]) + pu[2] * u[2]) + d[6];
  const double rl = ((u[0] * zeta[0] + u[1] * zeta[1]) + u[2] * zeta[2]) + vv[6];
  W[kWG] = wg;
  W[kV] = V;
  W[kRL] = rl;
  gg[e] = ((W[kP] + W[kP + 1]) + W[kP + 2]) - wg * wg / V;
  double g = (((vv[0] + vv[3]) + (vv[1] + vv[4])) + (vv[2] + vv[5])) - wg * rl / V;
  if (e == 0) g = g - 1.0;
  gr[e] = g;
  if (mode == 0) {
    const double* ze = z + kRows * (size_t)e;
    double* P = nrm + kNrm * (size_t)e;
    P[0] = pmax;
    P[1] = viol;
    P[2] = fabs(-(((u[0] * (ze[0] - ze[3]) + u[1] * (ze[1] - ze[4])) + u[2] * (ze[2] - ze[5]))) - ze[6]);
    P[3] = zg;
    P[4] = sz;
    P[5] = ze[6];
  }
}

// Owner CTA per free view a = blockIdx.x + 1 (rows 3 (a - 1) .. + 2), its incident edges in neighbour order.  mode 0:
// its off-diagonal blocks, its diagonal block and its entries of the gamma row (N - 1) into the zeroed N x N matrix,
// the max |dual residual| of its 3 coordinates into rdT[a - 1]; both modes: its right-hand side rows into
// rhs[stride * row].
__global__ void __launch_bounds__(128) k_tl_system(int mode, const uint32_t* __restrict__ inc_ofs, const uint32_t* __restrict__ inc_nbr,
                                                   const uint32_t* __restrict__ inc_edge, const uint2* __restrict__ ab,
                                                   const double* __restrict__ Rij, const double* __restrict__ ew,
                                                   const double* __restrict__ z, uint32_t N, double* __restrict__ A,
                                                   double* __restrict__ rhs, int stride, double* __restrict__ rdT) {
  const uint32_t a = blockIdx.x + 1, tid = threadIdx.x;
  const uint32_t ra_ = 3 * (a - 1);
  const uint32_t b0 = inc_ofs[a], b1 = inc_ofs[a + 1];
  if (mode == 0) {
    for (uint32_t p = b0 + tid; p < b1; p += blockDim.x) {
      const uint32_t e = inc_edge[p], b = inc_nbr[p];
      if (b == 0) continue;
      const double* R = Rij + 9 * (size_t)e;
      const double* W = ew + kEW * (size_t)e;
      const bool first = ab[e].x == a;  // a is the edge's I
      const double* wa = W + (first ? kWI : kWJ);
      const double* wb = W + (first ? kWJ : kWI);
      const double V = W[kV];
      for (int k = 0; k < 3; ++k)
        for (int l = 0; l < 3; ++l) {
          const double g = first ? -(R[3 * l + k] * W[kP + l]) : -(W[kP + k] * R[3 * k + l]);
          A[(size_t)(ra_ + k) * N + 3 * (b - 1) + l] = g - wa[k] * wb[l] / V;
        }
    }
  }
  if (tid < 9 && mode == 0) {  // diagonal block
    const int k = (int)tid / 3, l = (int)tid % 3;
    double acc = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const double* R = Rij + 9 * (size_t)e;
      const double* W = ew + kEW * (size_t)e;
      double t;
      const double* wa;
      if (ab[e].x == a) {
        t = ((R[k] * W[kP]) * R[l] + (R[3 + k] * W[kP + 1]) * R[3 + l]) + (R[6 + k] * W[kP + 2]) * R[6 + l];
        wa = W + kWI;
      } else {
        t = k == l ? W[kP + k] : 0.0;
        wa = W + kWJ;
      }
      acc += t - wa[k] * wa[l] / W[kV];
    }
    A[(size_t)(ra_ + k) * N + ra_ + l] = acc;
  } else if (tid >= 9 && tid < 12 && mode == 0) {  // the gamma row
    const int k = (int)tid - 9;
    double acc = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const double* R = Rij + 9 * (size_t)e;
      const double* W = ew + kEW * (size_t)e;
      double t;
      if (ab[e].x == a) {
        t = (R[k] * W[kQ] + R[3 + k] * W[kQ + 1]) + R[6 + k] * W[kQ + 2] - W[kWG] * W[kWI + k] / W[kV];
      } else {
        t = -W[kQ + k] - W[kWG] * W[kWJ + k] / W[kV];
      }
      acc += t;
    }
    A[(size_t)(N - 1) * N + ra_ + k] = acc;
  } else if (tid >= 12 && tid < 15) {  // the right-hand side
    const int k = (int)tid - 12;
    double acc = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const double* R = Rij + 9 * (size_t)e;
      const double* W = ew + kEW * (size_t)e;
      double t;
      if (ab[e].x == a) {
        t = ((R[k] * W[kZeta] + R[3 + k] * W[kZeta + 1]) + R[6 + k] * W[kZeta + 2]) - W[kWI + k] * W[kRL] / W[kV];
      } else {
        t = -W[kZeta + k] - W[kWJ + k] * W[kRL] / W[kV];
      }
      acc += t;
    }
    rhs[(size_t)stride * (ra_ + k)] = acc;
  } else if (tid == 15 && mode == 0) {  // the dual residual G^T z of the view's coordinates
    double acc[3] = {0.0, 0.0, 0.0};
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const double* R = Rij + 9 * (size_t)e;
      const double* ze = z + kRows * (size_t)e;
      const double zt[3] = {ze[0] - ze[3], ze[1] - ze[4], ze[2] - ze[5]};
      for (int k = 0; k < 3; ++k)
        acc[k] += ab[e].x == a ? -((R[k] * zt[0] + R[3 + k] * zt[1]) + R[6 + k] * zt[2]) : zt[k];
    }
    rdT[a - 1] = fmax(fmax(fabs(acc[0]), fabs(acc[1])), fabs(acc[2]));
  }
}

// out[0] = max |rp|, out[1] = max(0, G y - h), out[2] = max |G^T z + c|, out[3] = s^T z, out[4] = sum of z_lambda (the
// dual objective -h^T z)
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_tl_norms(const double* __restrict__ nrm, const double* __restrict__ rdT, uint32_t ne,
                                                       uint32_t nv, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double pm = 0.0, vi = 0.0, dm = 0.0, zg = 0.0, sz = 0.0, zl = 0.0;
  for (uint32_t e = threadIdx.x; e < ne; e += kThreads) {
    const double* P = nrm + kNrm * (size_t)e;
    pm = fmax(pm, P[0]);
    vi = fmax(vi, P[1]);
    dm = fmax(dm, P[2]);
    zg += P[3];
    sz += P[4];
    zl += P[5];
  }
  for (uint32_t v = threadIdx.x; v < nv; v += kThreads) dm = fmax(dm, rdT[v]);
  pm = block_max_fixed<kThreads>(pm, red);
  vi = block_max_fixed<kThreads>(vi, red);
  dm = block_max_fixed<kThreads>(dm, red);
  zg = block_sum_fixed<kThreads>(zg, red);
  sz = block_sum_fixed<kThreads>(sz, red);
  zl = block_sum_fixed<kThreads>(zl, red);
  if (threadIdx.x == 0) {
    out[0] = pm;
    out[1] = vi;
    out[2] = fmax(dm, fabs(1.0 - zg));
    out[3] = sz;
    out[4] = zl;
  }
}

// Per edge, from the reduced solution dy (T then gamma, stride apart): d lambda = (rhs_lambda - w^T dy) / V, the row
// steps G dy, ds = -rp - G dy, dz = wt + D G dy; ratio[2 e] = max(0, max -ds / s), ratio[2 e + 1] = the same for z.
__global__ void k_tl_back(const uint2* __restrict__ ab, const double* __restrict__ Rij, const double* __restrict__ uij,
                          const double* __restrict__ ew, const double* __restrict__ s, const double* __restrict__ z,
                          const double* __restrict__ dy, int stride, uint32_t ne, uint32_t N, double* __restrict__ dlam,
                          double* __restrict__ ds, double* __restrict__ dz, double* __restrict__ ratio) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  const double* R = Rij + 9 * (size_t)e;
  const double* u = uij + 3 * (size_t)e;
  const double* W = ew + kEW * (size_t)e;
  double TI[3], TJ[3];
  for (int k = 0; k < 3; ++k) {
    TI[k] = v.x == 0 ? 0.0 : dy[(size_t)stride * (3 * (v.x - 1) + k)];
    TJ[k] = v.y == 0 ? 0.0 : dy[(size_t)stride * (3 * (v.y - 1) + k)];
  }
  const double dg = dy[(size_t)stride * (N - 1)];
  const double wdy = (((W[kWI] * TI[0] + W[kWI + 1] * TI[1]) + W[kWI + 2] * TI[2]) + ((W[kWJ] * TJ[0] + W[kWJ + 1] * TJ[1]) + W[kWJ + 2] * TJ[2])) +
                     W[kWG] * dg;
  const double dl = (W[kRL] - wdy) / W[kV];
  dlam[e] = dl;
  double r[3], gd[kRows];
  edge_residual(R, u, TI, TJ, dl, r);
  for (int k = 0; k < 3; ++k) {
    gd[k] = r[k] - dg;
    gd[3 + k] = -r[k] - dg;
  }
  gd[6] = -dl;
  double ms = 0.0, mz = 0.0;
  for (int i = 0; i < kRows; ++i) {
    const double si = s[kRows * (size_t)e + i], zi = z[kRows * (size_t)e + i];
    const double dsi = -W[kRp + i] - gd[i];
    const double dzi = W[kWt + i] + (zi / si) * gd[i];
    ds[kRows * (size_t)e + i] = dsi;
    dz[kRows * (size_t)e + i] = dzi;
    ms = fmax(ms, -dsi / si);
    mz = fmax(mz, -dzi / zi);
  }
  ratio[2 * (size_t)e] = ms;
  ratio[2 * (size_t)e + 1] = mz;
}

// The step lengths alpha = min(1, eta / max ratio) for s (out[0]) and z (out[1]); mode 0 (predictor, eta = 1) also
// out[2] = (s + alpha_p ds)^T (z + alpha_d dz).
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_tl_ratio(int mode, const double* __restrict__ ratio, const double* __restrict__ s,
                                                       const double* __restrict__ z, const double* __restrict__ ds,
                                                       const double* __restrict__ dz, uint32_t ne, double eta, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double ms = 0.0, mz = 0.0;
  for (uint32_t e = threadIdx.x; e < ne; e += kThreads) {
    ms = fmax(ms, ratio[2 * (size_t)e]);
    mz = fmax(mz, ratio[2 * (size_t)e + 1]);
  }
  ms = block_max_fixed<kThreads>(ms, red);
  mz = block_max_fixed<kThreads>(mz, red);
  const double ap = ms > eta ? eta / ms : 1.0;
  const double ad = mz > eta ? eta / mz : 1.0;
  if (mode == 0) {
    double acc = 0.0;
    for (size_t i = threadIdx.x; i < kRows * (size_t)ne; i += kThreads) acc += (s[i] + ap * ds[i]) * (z[i] + ad * dz[i]);
    acc = block_sum_fixed<kThreads>(acc, red);
    if (threadIdx.x == 0) out[2] = acc;
  }
  if (threadIdx.x == 0) {
    out[0] = ap;
    out[1] = ad;
  }
}

// y += alpha_p dy (T and gamma), lambda += alpha_p d lambda, s += alpha_p ds, z += alpha_d dz; alpha from k_tl_ratio
__global__ void k_tl_update(const double* __restrict__ alpha, const double* __restrict__ dy, int stride, const double* __restrict__ dlam,
                            const double* __restrict__ ds, const double* __restrict__ dz, uint32_t ne, uint32_t N, double* __restrict__ y,
                            double* __restrict__ lam, double* __restrict__ s, double* __restrict__ z) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const double ap = alpha[0], ad = alpha[1];
  if (i < N) y[i] = y[i] + ap * dy[(size_t)stride * i];
  if (i >= ne) return;
  lam[i] = lam[i] + ap * dlam[i];
  for (int k = 0; k < kRows; ++k) {
    s[kRows * (size_t)i + k] = s[kRows * (size_t)i + k] + ap * ds[kRows * (size_t)i + k];
    z[kRows * (size_t)i + k] = z[kRows * (size_t)i + k] + ad * dz[kRows * (size_t)i + k];
  }
}

// the fallback of a failed factorisation: every diagonal entry of the N x N system += rel * its largest
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_tl_regularize(double* __restrict__ A, uint32_t N, double rel) {
  __shared__ double red[kThreads / 32];
  double m = 0.0;
  for (uint32_t i = threadIdx.x; i < N; i += kThreads) m = fmax(m, A[(size_t)i * N + i]);
  m = block_max_fixed<kThreads>(m, red);
  const double delta = rel * m;
  for (uint32_t i = threadIdx.x; i < N; i += kThreads) A[(size_t)i * N + i] = A[(size_t)i * N + i] + delta;
}

// Jacobi scaling of the assembled system: sc_i = 1 / sqrt(A_ii) (1 where A_ii <= 0)
__global__ void k_tl_jacobi_sc(const double* __restrict__ A, uint32_t N, double* __restrict__ sc) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double d = A[(size_t)i * N + i];
  sc[i] = d > 0.0 ? 1.0 / ::sqrt(d) : 1.0;
}

// one CTA per row i: A_ij <- (A_ij sc_i) sc_j, its copy into M (N x N); the right-hand side (row N of A) <- rhs_i sc_i,
// its copy into b
__global__ void k_tl_jacobi(double* __restrict__ A, uint32_t N, const double* __restrict__ sc, double* __restrict__ M,
                            double* __restrict__ b) {
  const uint32_t i = blockIdx.x;
  const double si = sc[i];
  for (uint32_t j = threadIdx.x; j < N; j += blockDim.x) {
    const double v = (A[(size_t)i * N + j] * si) * sc[j];
    A[(size_t)i * N + j] = v;
    M[(size_t)i * N + j] = v;
  }
  if (threadIdx.x == 0) {
    const double v = A[(size_t)N * N + i] * si;
    A[(size_t)N * N + i] = v;
    b[i] = v;
  }
}

// one warp per row i: Y[3 i] = b_i - (M x)_i with the symmetric M read from its lower triangle (lane-strided products,
// a fixed shuffle tree), Y[3 i + 1] = Y[3 i + 2] = 0
__global__ void k_tl_resid(const double* __restrict__ M, const double* __restrict__ b, const double* __restrict__ x, uint32_t N,
                           double* __restrict__ Y) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (i >= N) return;
  double acc = 0.0;
  for (uint32_t j = lane; j < N; j += 32) acc += (j <= i ? M[(size_t)i * N + j] : M[(size_t)j * N + i]) * x[j];
  for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    Y[3 * (size_t)i] = b[i] - acc;
    Y[3 * (size_t)i + 1] = 0.0;
    Y[3 * (size_t)i + 2] = 0.0;
  }
}

// mode 0: b_i = sc_i Y[3 i], Y[3 i] = b_i (the corrector's scaled right-hand side); mode 1: x_i = Y[3 i]; mode 2:
// x_i = sc_i (x_i + Y[3 i]) (the refined solution, unscaled)
__global__ void k_tl_vec(int mode, uint32_t N, const double* __restrict__ sc, double* __restrict__ Y, double* __restrict__ x,
                         double* __restrict__ b) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (mode == 0) {
    const double v = sc[i] * Y[3 * (size_t)i];
    b[i] = v;
    Y[3 * (size_t)i] = v;
  } else if (mode == 1) {
    x[i] = Y[3 * (size_t)i];
  } else {
    x[i] = sc[i] * (x[i] + Y[3 * (size_t)i]);
  }
}

// The start point, packed as a state (y: T of the free views then gamma, lambda, s, z; the last three in kept-edge
// order): T = 0, lambda = 2, gamma = 3 (strictly feasible: |u| = 1), s = h - G y, z = 1
std::vector<double> start_point(const ta::KeptEdges& K, uint32_t N) {
  const uint32_t ne = (uint32_t)K.kab.size();
  const size_t nr = (size_t)kRows * ne;
  std::vector<double> x(N + ne + 2 * nr, 0.0);
  x[N - 1] = 3.0;
  double* lam = x.data() + N;
  double* s = lam + ne;
  double* z = s + nr;
  for (uint32_t e = 0; e < ne; ++e) {
    lam[e] = 2.0;
    for (int k = 0; k < 3; ++k) {
      const double r = -2.0 * K.u[3 * (size_t)e + k];
      s[kRows * (size_t)e + k] = -(r - 3.0);
      s[kRows * (size_t)e + 3 + k] = -(-r - 3.0);
    }
    s[kRows * (size_t)e + 6] = 1.0;
  }
  for (size_t i = 0; i < nr; ++i) z[i] = 1.0;
  return x;
}

// The device side of one interior-point solve on the kept edges: its buffers and the four phases of an iteration.
// translation_averaging_l1 runs the phases back to back; r3d_debug_transavg_l1_step runs them once and reads the
// buffers back between them.
struct Ipm {
  r3d_ctx* ctx;
  DeviceWorker& w;
  const uint32_t m, ne, N;
  const size_t nr;
  const uint32_t eg, ug, vg;
  DevArr<uint32_t> d_iofs, d_inbr, d_iedge;
  DevArr<uint2> d_ab;
  DevArr<double> d_R, d_u, d_y, d_lam, d_s, d_z, d_ds, d_dz, d_dlam, d_ew, d_gg, d_gr, d_nrm, d_ratio, d_rdT, d_A, d_M, d_b, d_sc,
      d_L, d_Linv, d_x, d_Y, d_Z, d_scal;
  int trsm_grid = 0;
  // 0..4 k_tl_norms, 5 not-positive-definite flag, 8..10 k_tl_ratio, 15 gamma
  double h_scal[16] = {};
  int not_pd[kRegTries + 1] = {};  // the predictor's factorisation attempts
  uint32_t retries = 0;
  double sigma = 0.0;

  Ipm(r3d_ctx* c, DeviceWorker& wk, const ta::KeptEdges& K)
      : ctx(c), w(wk), m((uint32_t)K.kview.size()), ne((uint32_t)K.kab.size()), N(3 * (m - 1) + 1), nr((size_t)kRows * ne),
        eg((ne + 127) / 128), ug((std::max(ne, N) + 127) / 128), vg((N + 127) / 128), d_iofs(wk), d_inbr(wk), d_iedge(wk), d_ab(wk),
        d_R(wk), d_u(wk), d_y(wk), d_lam(wk), d_s(wk), d_z(wk), d_ds(wk), d_dz(wk), d_dlam(wk), d_ew(wk), d_gg(wk), d_gr(wk), d_nrm(wk),
        d_ratio(wk), d_rdT(wk), d_A(wk), d_M(wk), d_b(wk), d_sc(wk), d_L(wk), d_Linv(wk), d_x(wk), d_Y(wk), d_Z(wk), d_scal(wk) {}

  // the scratch, the kept edges and their incidence lists on the device, the state x (packed as start_point's)
  int init(const char* fn, const ta::KeptEdges& K, const std::vector<double>& x) {
    std::vector<uint32_t> inc_ofs, inc_nbr, inc_edge;
    ra::incidence_lists(m, K.kab, inc_ofs, inc_nbr, inc_edge);
    const int nblk = ((int)N + kCholNB - 1) / kCholNB;
    if (!d_iofs.alloc(m + 1) || !d_inbr.alloc(2 * (size_t)ne) || !d_iedge.alloc(2 * (size_t)ne) || !d_ab.alloc(ne) || !d_R.alloc(9 * (size_t)ne) ||
        !d_u.alloc(3 * (size_t)ne) || !d_y.alloc(N) || !d_lam.alloc(ne) || !d_s.alloc(nr) || !d_z.alloc(nr) || !d_ds.alloc(nr) ||
        !d_dz.alloc(nr) || !d_dlam.alloc(ne) || !d_ew.alloc((size_t)kEW * ne) || !d_gg.alloc(ne) || !d_gr.alloc(ne) ||
        !d_nrm.alloc((size_t)kNrm * ne) || !d_ratio.alloc(2 * (size_t)ne) || !d_rdT.alloc(m - 1) || !d_A.alloc((size_t)(N + 1) * N) ||
        !d_L.alloc((size_t)(N + 1) * N + 64) || !d_Linv.alloc((size_t)nblk * kCholNB * kCholNB) || !d_x.alloc(N) ||
        !d_Y.alloc(3 * (size_t)N) || !d_Z.alloc(3 * (size_t)N) || !d_M.alloc((size_t)N * N) || !d_b.alloc(N) || !d_sc.alloc(N) ||
        !d_scal.alloc(16))
      return fail(ctx, R3D_ERR_NOMEM, std::string(fn) + "device scratch");
    R3D_CUDA_TRY(ctx, h2d(d_iofs.p, inc_ofs.data(), (m + 1) * sizeof(uint32_t)));
    R3D_CUDA_TRY(ctx, h2d(d_inbr.p, inc_nbr.data(), inc_nbr.size() * sizeof(uint32_t)));
    R3D_CUDA_TRY(ctx, h2d(d_iedge.p, inc_edge.data(), inc_edge.size() * sizeof(uint32_t)));
    R3D_CUDA_TRY(ctx, h2d(d_ab.p, K.ab.data(), ne * sizeof(uint2)));
    R3D_CUDA_TRY(ctx, h2d(d_R.p, K.Rij.data(), K.Rij.size() * sizeof(double)));
    R3D_CUDA_TRY(ctx, h2d(d_u.p, K.u.data(), K.u.size() * sizeof(double)));
    R3D_CUDA_TRY(ctx, h2d(d_y.p, x.data(), N * sizeof(double)));
    R3D_CUDA_TRY(ctx, h2d(d_lam.p, x.data() + N, ne * sizeof(double)));
    R3D_CUDA_TRY(ctx, h2d(d_s.p, x.data() + N + ne, nr * sizeof(double)));
    R3D_CUDA_TRY(ctx, h2d(d_z.p, x.data() + N + ne + nr, nr * sizeof(double)));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_scal.p, 0, 16 * sizeof(double), w.stream));
    return ra::trsm3_grid(ctx, w, &trsm_grid);
  }

  cudaError_t h2d(void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, w.stream); }

  int read_scal() {
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(h_scal, d_scal.p, sizeof(h_scal), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    return R3D_OK;
  }

  // one step of iterative refinement of the scaled solution in d_x against the unregularised M, b, then unscaled:
  // x <- sc (x + (L L^T)^-1 (b - M x))
  int refine() {
    k_tl_resid<<<(N + 3) / 4, 128, 0, w.stream>>>(d_M.p, d_b.p, d_x.p, N, d_Y.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    int rc;
    if ((rc = ra::trsm3(ctx, w, d_L.p, d_Linv.p, (int)N, d_Y.p, d_Z.p, trsm_grid))) return rc;
    k_tl_vec<<<vg, 128, 0, w.stream>>>(2, N, d_sc.p, d_Y.p, d_x.p, d_b.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return R3D_OK;
  }

  // phase 1: the residuals, the reduced system of the current point (the matrix and the predictor's right-hand side
  // into d_A, unscaled) and the norms (h_scal 0..4, gamma in h_scal 15)
  int assemble() {
    k_tl_rows<<<eg, 128, 0, w.stream>>>(0, d_ab.p, d_R.p, d_u.p, d_y.p, d_lam.p, d_s.p, d_z.p, d_ds.p, d_dz.p, 0.0, ne, N, d_ew.p,
                                        d_gg.p, d_gr.p, d_nrm.p);
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_A.p, 0, (size_t)(N + 1) * N * sizeof(double), w.stream));
    k_tl_system<<<m - 1, 128, 0, w.stream>>>(0, d_iofs.p, d_inbr.p, d_iedge.p, d_ab.p, d_R.p, d_ew.p, d_z.p, N, d_A.p,
                                             d_A.p + (size_t)N * N, 1, d_rdT.p);
    ra::k_avg_sum<ra::kAvgThreads><<<1, ra::kAvgThreads, 0, w.stream>>>(d_gg.p, ne, d_A.p + (size_t)(N - 1) * N + (N - 1));
    ra::k_avg_sum<ra::kAvgThreads><<<1, ra::kAvgThreads, 0, w.stream>>>(d_gr.p, ne, d_A.p + (size_t)N * N + (N - 1));
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    k_tl_norms<ra::kAvgThreads><<<1, ra::kAvgThreads, 0, w.stream>>>(d_nrm.p, d_rdT.p, ne, m - 1, d_scal.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_scal.p + 15, d_y.p + (N - 1), sizeof(double), cudaMemcpyDeviceToDevice, w.stream));
    return read_scal();
  }

  // the stopping test on phase 1's norms (|h|_inf = 1)
  bool converged(double tol) const {
    const double pres = h_scal[0], dres = h_scal[2], dobj = h_scal[4], gam = h_scal[15];
    return pres <= tol * 2.0 && dres <= tol && std::fabs(gam - dobj) <= tol * (1.0 + std::fabs(gam));
  }

  // one factorisation attempt (reg > 0: of M + reg max(diag) I, from the copy), its solve refined against M, the step
  // lengths and the complementarity they reach
  int predictor_attempt(double reg) {
    if (reg > 0.0) {
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_A.p, d_M.p, (size_t)N * N * sizeof(double), cudaMemcpyDeviceToDevice, w.stream));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_A.p + (size_t)N * N, d_b.p, N * sizeof(double), cudaMemcpyDeviceToDevice, w.stream));
      k_tl_regularize<kRThreads><<<1, kRThreads, 0, w.stream>>>(d_A.p, N, reg);
    }
    double* scal = d_scal.p;
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(scal + 5, 0, sizeof(double), w.stream));
    int rc;
    if ((rc = dense_cholesky(ctx, w, d_A.p, d_L.p, d_Linv.p, (int)N, scal + 5, d_x.p))) return rc;
    if ((rc = refine())) return rc;
    k_tl_back<<<eg, 128, 0, w.stream>>>(d_ab.p, d_R.p, d_u.p, d_ew.p, d_s.p, d_z.p, d_x.p, 1, ne, N, d_dlam.p, d_ds.p, d_dz.p, d_ratio.p);
    k_tl_ratio<kRThreads><<<1, kRThreads, 0, w.stream>>>(0, d_ratio.p, d_s.p, d_z.p, d_ds.p, d_dz.p, ne, 1.0, scal + 8);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return read_scal();
  }

  // phase 2: the system scaled to a unit diagonal (M, b: the unregularised copy), the predictor, and while its
  // factorisation is not positive definite, again with the diagonal raised.  *failed: every attempt failed.
  int predictor(bool* failed) {
    k_tl_jacobi_sc<<<(N + 127) / 128, 128, 0, w.stream>>>(d_A.p, N, d_sc.p);
    k_tl_jacobi<<<N, 128, 0, w.stream>>>(d_A.p, N, d_sc.p, d_M.p, d_b.p);
    std::fill(not_pd, not_pd + kRegTries + 1, 0);
    retries = 0;
    int rc;
    if ((rc = predictor_attempt(0.0))) return rc;
    not_pd[0] = h_scal[5] != 0.0;
    double reg = kRegRel;
    for (int k = 0; k < kRegTries && h_scal[5] != 0.0; ++k, reg *= kRegGrowth) {
      ++retries;
      if ((rc = predictor_attempt(reg))) return rc;
      not_pd[k + 1] = h_scal[5] != 0.0;
    }
    *failed = h_scal[5] != 0.0;
    return R3D_OK;
  }

  // phase 3: sigma = (mu_aff / mu)^3, the corrector through the predictor's factor: the right-hand side with the
  // predictor's second-order term and sigma mu, its solve refined against M, the step lengths (h_scal 8, 9 after the
  // next read)
  int corrector() {
    const double nrows = (double)nr;
    const double mu = h_scal[3] / nrows, ratio_mu = (h_scal[10] / nrows) / mu;
    sigma = (ratio_mu * ratio_mu) * ratio_mu;
    k_tl_rows<<<eg, 128, 0, w.stream>>>(1, d_ab.p, d_R.p, d_u.p, d_y.p, d_lam.p, d_s.p, d_z.p, d_ds.p, d_dz.p, sigma * mu, ne, N,
                                        d_ew.p, d_gg.p, d_gr.p, d_nrm.p);
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_Y.p, 0, 3 * (size_t)N * sizeof(double), w.stream));
    k_tl_system<<<m - 1, 128, 0, w.stream>>>(1, d_iofs.p, d_inbr.p, d_iedge.p, d_ab.p, d_R.p, d_ew.p, d_z.p, N, d_A.p, d_Y.p, 3,
                                             d_rdT.p);
    ra::k_avg_sum<ra::kAvgThreads><<<1, ra::kAvgThreads, 0, w.stream>>>(d_gr.p, ne, d_Y.p + 3 * (size_t)(N - 1));
    k_tl_vec<<<vg, 128, 0, w.stream>>>(0, N, d_sc.p, d_Y.p, d_x.p, d_b.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    int rc;
    if ((rc = ra::trsm3(ctx, w, d_L.p, d_Linv.p, (int)N, d_Y.p, d_Z.p, trsm_grid))) return rc;
    k_tl_vec<<<vg, 128, 0, w.stream>>>(1, N, d_sc.p, d_Y.p, d_x.p, d_b.p);
    if ((rc = refine())) return rc;
    k_tl_back<<<eg, 128, 0, w.stream>>>(d_ab.p, d_R.p, d_u.p, d_ew.p, d_s.p, d_z.p, d_x.p, 1, ne, N, d_dlam.p, d_ds.p, d_dz.p, d_ratio.p);
    k_tl_ratio<kRThreads><<<1, kRThreads, 0, w.stream>>>(1, d_ratio.p, d_s.p, d_z.p, d_ds.p, d_dz.p, ne, kEta, d_scal.p + 8);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return R3D_OK;
  }

  // phase 4: the step
  int update() {
    k_tl_update<<<ug, 128, 0, w.stream>>>(d_scal.p + 8, d_x.p, 1, d_dlam.p, d_ds.p, d_dz.p, ne, N, d_y.p, d_lam.p, d_s.p, d_z.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return R3D_OK;
  }
};

int translation_averaging_l1(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use, const double* rot,
                             const uint8_t* rot_kept, uint32_t n_views, const r3d_transavg_l1_options& opt, double* centers,
                             double* translations, uint8_t* view_kept, uint8_t* edge_kept, double* edge_scale,
                             r3d_transavg_l1_summary& S) {
  const double t0 = now_ms();
  const char* fn = "r3d_translation_averaging_l1: ";
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::memset(centers, 0, (size_t)n_views * 3 * sizeof(double));
  std::memset(translations, 0, (size_t)n_views * 3 * sizeof(double));
  std::memset(view_kept, 0, n_views);
  if (edge_kept) std::memset(edge_kept, 0, n_rel);
  if (edge_scale) std::memset(edge_scale, 0, n_rel * sizeof(double));
  // ---- 1. the kept edges (transavg.cu) ----
  ta::KeptEdges K;
  int rc = ta::select_edges(ctx, fn, rel, n_rel, edge_use, rot, rot_kept, n_views, K);
  S.n_edges = K.n_edges;
  if (rc) return rc;
  if (K.kview.empty()) {
    S.ms_host = now_ms() - t0;
    return R3D_OK;
  }
  const uint32_t m = (uint32_t)K.kview.size(), ne = (uint32_t)K.kab.size();
  S.success = 1;
  S.n_kept_views = m;
  S.n_kept_edges = ne;
  for (uint32_t v : K.kview) view_kept[v] = 1;
  if (edge_kept)
    for (uint64_t src : K.src) edge_kept[src] = 1;
  // ---- 2. the interior-point method ----
  Ipm P(ctx, w, K);
  const uint32_t N = P.N;  // free view translations, then gamma
  if ((rc = P.init(fn, K, start_point(K, N)))) return rc;
  Events<2> evt;
  R3D_CUDA_TRY(ctx, evt.create());
  R3D_CUDA_TRY(ctx, cudaEventRecord(evt.e[0], w.stream));
  int term = 1;
  uint32_t it = 0, nreg = 0;
  for (;; ++it) {
    if ((rc = P.assemble())) return rc;
    if (P.converged(opt.tolerance)) {
      term = 0;
      break;
    }
    if (it == (uint32_t)opt.max_iterations) break;
    bool failed = false;
    if ((rc = P.predictor(&failed))) return rc;
    nreg += P.retries;
    if (failed) {
      term = 2;
      break;
    }
    if ((rc = P.corrector()) || (rc = P.update())) return rc;
  }
  std::vector<double> y(N), lam(ne);
  R3D_CUDA_TRY(ctx, cudaEventRecord(evt.e[1], w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(y.data(), P.d_y.p, N * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(lam.data(), P.d_lam.p, ne * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  S.ms_solve = evt.ms(0, 1);
  S.iterations = it;
  S.regularized_factorizations = nreg;
  S.termination = term;
  S.gamma = P.h_scal[15];
  S.dual_objective = P.h_scal[4];
  S.max_primal_violation = P.h_scal[1];
  S.max_dual_violation = P.h_scal[2];
  // translations T (the lowest kept view: 0), centres C = -R^T T, the scales of the kept edges
  for (uint32_t a = 0; a < m; ++a) {
    const uint32_t v = K.kview[a];
    const double* R = rot + 9 * (size_t)v;
    double p[3];
    for (int k = 0; k < 3; ++k) p[k] = a == 0 ? 0.0 : y[3 * (size_t)(a - 1) + k];
    for (int k = 0; k < 3; ++k) {
      translations[3 * (size_t)v + k] = p[k];
      centers[3 * (size_t)v + k] = -(R[k] * p[0] + R[3 + k] * p[1] + R[6 + k] * p[2]);
    }
  }
  if (edge_scale)
    for (uint32_t e = 0; e < ne; ++e) edge_scale[K.src[e]] = lam[e];
  S.ms_device_total = S.ms_solve;
  S.ms_host = now_ms() - t0 - S.ms_device_total;
  return R3D_OK;
}

// r3d_debug_transavg_l1_step: one iteration of the phases above from the state x (or the start point)
int debug_step(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use, const double* rot,
               const uint8_t* rot_kept, uint32_t n_views, const double* state, uint64_t n_state, double tolerance,
               r3d_transavg_l1_step_out& O) {
  const char* fn = "r3d_debug_transavg_l1_step: ";
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  ta::KeptEdges K;
  int rc = ta::select_edges(ctx, fn, rel, n_rel, edge_use, rot, rot_kept, n_views, K);
  if (rc) return rc;
  if (K.kview.empty()) return R3D_OK;
  const uint32_t m = (uint32_t)K.kview.size(), ne = (uint32_t)K.kab.size(), N = 3 * (m - 1) + 1;
  const size_t nr = (size_t)kRows * ne, nx = N + ne + 2 * nr;
  std::vector<double> x;
  if (!state) {
    x = start_point(K, N);
  } else {
    if (n_state != nx) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "the state must hold N + 15 x kept edges values");
    x.assign(state, state + nx);
    for (size_t i = 0; i < nx; ++i)
      if (!std::isfinite(x[i])) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "a non-finite state");
    for (size_t i = 0; i < nr; ++i)
      if (!(x[N + ne + i] > 0.0) || !(x[N + ne + nr + i] >= 0.0)) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "s <= 0 or z < 0");
  }
  O.n_kept_views = m;
  O.n_kept_edges = ne;
  O.n = N;
  for (uint32_t a = 0; a < m; ++a)
    if (O.view_ids) O.view_ids[a] = K.kview[a];
  for (uint32_t e = 0; e < ne; ++e) {
    if (O.edge_record) O.edge_record[e] = K.src[e];
    if (O.edge_ij) {
      O.edge_ij[2 * (size_t)e] = K.ab[e].x;
      O.edge_ij[2 * (size_t)e + 1] = K.ab[e].y;
    }
  }
  if (O.Rij) std::memcpy(O.Rij, K.Rij.data(), K.Rij.size() * sizeof(double));
  if (O.u) std::memcpy(O.u, K.u.data(), K.u.size() * sizeof(double));
  if (O.state0) std::memcpy(O.state0, x.data(), nx * sizeof(double));
  Ipm P(ctx, w, K);
  if ((rc = P.init(fn, K, x))) return rc;
  auto d2h = [&](double* dst, const double* src, size_t n) -> int {
    if (dst) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(dst, src, n * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
    return R3D_OK;
  };
  auto d2h_sync = [&]() -> int {
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    return R3D_OK;
  };
  // the step of one phase: the direction of the reduced solve and its back-substitution
  auto direction = [&](double* dy, double* dlam, double* ds, double* dz) -> int {
    if ((rc = d2h(dy, P.d_x.p, N)) || (rc = d2h(dlam, P.d_dlam.p, ne)) || (rc = d2h(ds, P.d_ds.p, nr)) || (rc = d2h(dz, P.d_dz.p, nr)))
      return rc;
    return d2h_sync();
  };
  if ((rc = P.assemble())) return rc;
  std::memcpy(O.norms, P.h_scal, sizeof(O.norms));
  if ((rc = d2h(O.A, P.d_A.p, (size_t)(N + 1) * N)) || (rc = d2h_sync())) return rc;
  if (P.converged(tolerance)) {
    O.converged = 1;
    return R3D_OK;
  }
  bool failed = false;
  if ((rc = P.predictor(&failed))) return rc;
  std::copy(P.not_pd, P.not_pd + kRegTries + 1, O.not_pd);
  O.retries = P.retries;
  if ((rc = d2h(O.sc, P.d_sc.p, N)) || (rc = direction(O.pred_dy, O.pred_dlam, O.pred_ds, O.pred_dz))) return rc;
  O.pred_alpha_p = P.h_scal[8];
  O.pred_alpha_d = P.h_scal[9];
  O.pred_complementarity = P.h_scal[10];
  if (failed) {
    O.failed = 1;
    return R3D_OK;
  }
  if ((rc = P.corrector())) return rc;
  O.sigma = P.sigma;
  if ((rc = d2h(O.corr_rhs, P.d_b.p, N)) || (rc = direction(O.corr_dy, O.corr_dlam, O.corr_ds, O.corr_dz)) || (rc = P.read_scal()))
    return rc;
  O.alpha_p = P.h_scal[8];
  O.alpha_d = P.h_scal[9];
  if ((rc = P.update())) return rc;
  if (O.state) {
    if ((rc = d2h(O.state, P.d_y.p, N)) || (rc = d2h(O.state + N, P.d_lam.p, ne)) || (rc = d2h(O.state + N + ne, P.d_s.p, nr)) ||
        (rc = d2h(O.state + N + ne + nr, P.d_z.p, nr)))
      return rc;
  }
  return d2h_sync();
}

}  // namespace tl
}  // namespace r3d

using namespace r3d;

extern "C" void r3d_transavg_l1_default_options(r3d_transavg_l1_options* o) {
  if (!o) return;
  o->max_iterations = 100;
  o->tolerance = 1e-9;
}

extern "C" int r3d_translation_averaging_l1(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                                            const double* rotations, const uint8_t* rot_kept, uint32_t n_views,
                                            const r3d_transavg_l1_options* opt, double* centers, double* translations,
                                            uint8_t* view_kept, uint8_t* edge_kept, double* edge_scale,
                                            r3d_transavg_l1_summary* summary) {
  if (!ctx || (!rel && n_rel) || !opt || (n_views && (!rotations || !rot_kept || !centers || !translations || !view_kept)) || !summary)
    return fail(ctx, R3D_ERR_INVALID, "r3d_translation_averaging_l1: bad arguments");
  std::memset(summary, 0, sizeof(*summary));
  summary->termination = -1;
  if (opt->max_iterations < 1 || !(opt->tolerance > 0.0))
    return fail(ctx, R3D_ERR_INVALID, "r3d_translation_averaging_l1: max_iterations < 1 or tolerance <= 0");
  return tl::translation_averaging_l1(ctx, rel, n_rel, edge_use, rotations, rot_kept, n_views, *opt, centers, translations, view_kept,
                                      edge_kept, edge_scale, *summary);
}

extern "C" int r3d_debug_transavg_l1_step(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                                          const double* rotations, const uint8_t* rot_kept, uint32_t n_views, const double* state,
                                          uint64_t n_state, double tolerance, r3d_transavg_l1_step_out* out) {
  if (!ctx || (!rel && n_rel) || (n_views && (!rotations || !rot_kept)) || (!state && n_state) || !(tolerance > 0.0) || !out)
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_transavg_l1_step: bad arguments");
  r3d_transavg_l1_step_out& O = *out;
  O.n_kept_views = O.n_kept_edges = O.n = 0;
  std::memset(O.norms, 0, sizeof(O.norms));
  std::memset(O.not_pd, 0, sizeof(O.not_pd));
  O.retries = 0;
  O.pred_alpha_p = O.pred_alpha_d = O.pred_complementarity = O.sigma = O.alpha_p = O.alpha_d = 0.0;
  O.converged = O.failed = 0;
  return tl::debug_step(ctx, rel, n_rel, edge_use, rotations, rot_kept, n_views, state, n_state, tolerance, O);
}
