// rotavg_l1.cu -- global camera rotations by Chatterjee & Govindu's robust method (L1RA then IRLS), Regard3D's "L1
// rotation averaging" (r3d_rotation_averaging_l1).
// COMPILED WITH --fmad=false (regard3d_b200/build.py), like rotavg.cu: every product and sum is written out in one
// fixed order and no kernel uses floating-point atomics, so repeated calls are bit-identical.
//
// Steps 1 and 2 (edge checks, triplet rejection, the largest bi-edge-connected component) are rotavg.cu's
// select_component.  Then, on kept local ids (local 0 held at R = I), with R_b = R_ab R_a:
//   start   host: a breadth-first spanning tree from local 0, neighbours in ascending order
//   L1RA    per outer iteration k_l1_residual (b_e = log(R_b^T R_ab R_a), the Ceres quaternion log), then l1-magic's
//           l1decode_pd (Candes & Romberg) for x = argmin |A x - b|_1 from x = 0, then k_l1_rotate (R_v <- R_v exp(x_v))
//   IRLS    per iteration k_l1_residual, k_l1_irls (the weights), the weighted normal equations, k_l1_rotate
// A (3E x 3(m - 1)): row 3e + k holds -1 at (a, k) and +1 at (b, k).  Every row touches one component k, so
// A^T diag(d) A is three weighted graph Laplacians of size n = m - 1, one per component: k_l1_system assembles them
// (one owner CTA per view) and dense_cholesky (ba.cu) factors each.  Per-row data stays on the device; the host reads
// back only the scalars of one Newton step or one backtrack.
// Layouts: per-row arrays are E x 3 (row 3e + k); per-variable arrays are component-major (k n + a - 1).
#include "r3d_internal.cuh"
#include "averaging.cuh"
#include "detmath.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace r3d {
namespace rl {

// l1decode_pd's constants
constexpr double kPdTol = 1e-3;      // stop when the surrogate duality gap < kPdTol
constexpr int kPdMaxIter = 50;
constexpr double kPdMu = 10.0;
constexpr double kPdAlpha = 0.01;    // sufficient decrease of the residual norm
constexpr double kPdBeta = 0.5;      // backtracking factor
constexpr int kPdMaxBacktracks = 32;
constexpr int kRThreads = 1024;      // the one-CTA reductions

__device__ __forceinline__ double vcoord(const double* x, uint32_t n, uint32_t v, int k) { return v == 0 ? 0.0 : x[(size_t)k * n + v - 1]; }

// per kept edge: b = log(R_b^T (R_ab R_a)), cost[e] = |b|_1
__global__ void k_l1_residual(const double* __restrict__ R, const uint2* __restrict__ ab, const double* __restrict__ Rk, uint32_t ne,
                              double* __restrict__ b, double* __restrict__ cost) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  const double* Ra = R + 9 * (size_t)v.x;
  const double* Rb = R + 9 * (size_t)v.y;
  const double* Q = Rk + 9 * (size_t)e;
  double P[9], E[9], r[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) P[3 * i + j] = (Q[3 * i] * Ra[j] + Q[3 * i + 1] * Ra[3 + j]) + Q[3 * i + 2] * Ra[6 + j];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[3 * i + j] = (Rb[i] * P[j] + Rb[3 + i] * P[3 + j]) + Rb[6 + i] * P[6 + j];
  ra::R_to_aa(E, r);
  for (int k = 0; k < 3; ++k) b[3 * (size_t)e + k] = r[k];
  cost[e] = (fabs(r[0]) + fabs(r[1])) + fabs(r[2]);
}

// one thread per free view a = thread + 1: R_a <- R_a exp([x_a]x) (Ceres' angle-axis to matrix)
__global__ void k_l1_rotate(const double* __restrict__ x, uint32_t n, double* __restrict__ R) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const double aa[3] = {x[t], x[(size_t)n + t], x[2 * (size_t)n + t]};
  double Q[9], Rn[9];
  ra::aa_to_R(aa, Q);
  double* Ra = R + 9 * (size_t)(t + 1);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Rn[3 * i + j] = (Ra[3 * i] * Q[j] + Ra[3 * i + 1] * Q[3 + j]) + Ra[3 * i + 2] * Q[6 + j];
  for (int c = 0; c < 9; ++c) Ra[c] = Rn[c];
}

// One owner CTA per free view a = blockIdx.x + 1, its incident edges in neighbour order: row a - 1 of the three
// Laplacians of the row weights w (component k: A3 + k mstride, n x n, off-diagonal -w, diagonal the sum of w) and,
// with v, the right-hand sides (A^T v)_(a, k) into row n of each.  The caller zeroes A3.
__global__ void __launch_bounds__(128) k_l1_system(const uint32_t* __restrict__ inc_ofs, const uint32_t* __restrict__ inc_nbr,
                                                   const uint32_t* __restrict__ inc_edge, const uint2* __restrict__ ab,
                                                   const double* __restrict__ w, const double* __restrict__ v, uint32_t n,
                                                   size_t mstride, double* __restrict__ A3) {
  const uint32_t a = blockIdx.x + 1, tid = threadIdx.x;
  const uint32_t b0 = inc_ofs[a], b1 = inc_ofs[a + 1];
  for (uint32_t p = b0 + tid; p < b1; p += blockDim.x) {
    const uint32_t e = inc_edge[p], b = inc_nbr[p];
    if (b == 0) continue;
    for (int k = 0; k < 3; ++k) A3[k * mstride + (size_t)(a - 1) * n + b - 1] = -w[3 * (size_t)e + k];
  }
  if (tid < 3) {
    const int k = (int)tid;
    double s = 0.0;
    for (uint32_t p = b0; p < b1; ++p) s += w[3 * (size_t)inc_edge[p] + k];
    A3[k * mstride + (size_t)(a - 1) * n + a - 1] = s;
  } else if (tid < 6) {
    const int k = (int)tid - 3;
    double s = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const double t = v[3 * (size_t)e + k];
      s += ab[e].y == a ? t : -t;
    }
    A3[k * mstride + (size_t)n * n + a - 1] = s;
  }
}

// A^T v (component-major, n per component) of the row vector v: one thread per (free view, component), its incident
// edges in neighbour order
__global__ void k_l1_at(const uint32_t* __restrict__ inc_ofs, const uint32_t* __restrict__ inc_edge, const uint2* __restrict__ ab,
                        const double* __restrict__ v, uint32_t n, double* __restrict__ out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * n) return;
  const uint32_t a = t % n + 1;
  const int k = (int)(t / n);
  double s = 0.0;
  for (uint32_t p = inc_ofs[a]; p < inc_ofs[a + 1]; ++p) {
    const uint32_t e = inc_edge[p];
    const double x = v[3 * (size_t)e + k];
    s += ab[e].y == a ? x : -x;
  }
  out[t] = s;
}

// The primal-dual state of l1decode_pd: x (3n), A x, u, lambda_1, lambda_2 (3E each), A^T (lambda_1 - lambda_2) (3n).
// fu1 = (A x - b) - u, fu2 = (-A x + b) - u are formed where they are used.
struct PdState {
  double *x, *Ax, *u, *l1, *l2, *Atv;
};

// per row: the start u = 0.95 |b| + 0.1 max |b| (bmax = *bm), A x = 0, lambda = -1 / fu, dv = lambda_1 - lambda_2
__global__ void k_l1_pd_start(const double* __restrict__ b, const double* __restrict__ bm, uint32_t nr, PdState s, double* __restrict__ dv) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  const double bi = b[i];
  const double u = 0.95 * fabs(bi) + 0.10 * bm[0];
  const double f1 = (0.0 - bi) - u, f2 = (-0.0 + bi) - u;
  const double l1 = -1.0 / f1, l2 = -1.0 / f2;
  s.Ax[i] = 0.0;
  s.u[i] = u;
  s.l1[i] = l1;
  s.l2[i] = l2;
  dv[i] = l1 - l2;
}

// the terms of the residual norm and of the surrogate duality gap of one row and one variable
__device__ __forceinline__ void row_terms(double b, double Ax, double u, double l1, double l2, double tinv, double& res, double& sz) {
  const double f1 = (Ax - b) - u, f2 = (-Ax + b) - u;
  const double rd = (1.0 - l1) - l2;
  const double rc1 = -l1 * f1 - tinv, rc2 = -l2 * f2 - tinv;
  res += (rd * rd + rc1 * rc1) + rc2 * rc2;
  sz += f1 * l1 + f2 * l2;
}

// Over max(E, n) threads: thread t sums its edge's 3 rows (t < E) and its variable's 3 components (t < n) into
// part[t] (|rdual|^2 + |rcent|^2 with 1 / tau = tinv) and part[P + t] (sum fu^T lambda, the duality gap's negative).
__global__ void k_l1_norms(const double* __restrict__ b, PdState s, uint32_t ne, uint32_t n, double tinv, uint32_t P,
                           double* __restrict__ part) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= P) return;
  double res = 0.0, sz = 0.0;
  if (t < ne)
    for (int k = 0; k < 3; ++k) {
      const size_t i = 3 * (size_t)t + k;
      row_terms(b[i], s.Ax[i], s.u[i], s.l1[i], s.l2[i], tinv, res, sz);
    }
  if (t < n)
    for (int k = 0; k < 3; ++k) {
      const double g = s.Atv[(size_t)k * n + t];
      res += g * g;
    }
  part[t] = res;
  part[P + t] = sz;
}

// per row, the Newton system's row quantities: sigx (the Laplacians' weights), the right-hand side's row vector
// rrow = -(1/tau) (-1/fu1 + 1/fu2) - (sig2 / sig1) w2, and w2
__global__ void k_l1_newton(const double* __restrict__ b, PdState s, uint32_t nr, double tinv, double* __restrict__ sigx,
                            double* __restrict__ rrow, double* __restrict__ w2o) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  const double Ax = s.Ax[i], u = s.u[i], l1 = s.l1[i], l2 = s.l2[i], bi = b[i];
  const double f1 = (Ax - bi) - u, f2 = (-Ax + bi) - u;
  const double w2 = -1.0 - tinv * (1.0 / f1 + 1.0 / f2);
  const double sig1 = -l1 / f1 - l2 / f2;
  const double sig2 = l1 / f1 - l2 / f2;
  sigx[i] = sig1 - sig2 * sig2 / sig1;
  rrow[i] = -tinv * (-1.0 / f1 + 1.0 / f2) - (sig2 / sig1) * w2;
  w2o[i] = w2;
}

// The direction of the other unknowns from dx (component-major), per edge and its 3 rows: A dx, du, d lambda_1,
// d lambda_2, dv = d lambda_1 - d lambda_2, and rmin[e] = min(1, the largest steps that keep lambda > 0 and fu < 0)
struct PdDir {
  double *Adx, *du, *dl1, *dl2;
};
__global__ void k_l1_direction(const uint2* __restrict__ ab, const double* __restrict__ b, PdState s, const double* __restrict__ w2,
                               const double* __restrict__ dx, uint32_t ne, uint32_t n, double tinv, PdDir d, double* __restrict__ dv,
                               double* __restrict__ rmin) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  double r = 1.0;
  for (int k = 0; k < 3; ++k) {
    const size_t i = 3 * (size_t)e + k;
    const double Ax = s.Ax[i], u = s.u[i], l1 = s.l1[i], l2 = s.l2[i], bi = b[i];
    const double f1 = (Ax - bi) - u, f2 = (-Ax + bi) - u;
    const double sig1 = -l1 / f1 - l2 / f2;
    const double sig2 = l1 / f1 - l2 / f2;
    const double adx = vcoord(dx, n, v.y, k) - vcoord(dx, n, v.x, k);
    const double du = (w2[i] - sig2 * adx) / sig1;
    const double dl1 = -(l1 / f1) * (adx - du) - l1 - tinv / f1;
    const double dl2 = (l2 / f2) * (adx + du) - l2 - tinv / f2;
    d.Adx[i] = adx;
    d.du[i] = du;
    d.dl1[i] = dl1;
    d.dl2[i] = dl2;
    dv[i] = dl1 - dl2;
    if (dl1 < 0.0) r = fmin(r, -l1 / dl1);
    if (dl2 < 0.0) r = fmin(r, -l2 / dl2);
    const double g1 = adx - du, g2 = -adx - du;
    if (g1 > 0.0) r = fmin(r, -f1 / g1);
    if (g2 > 0.0) r = fmin(r, -f2 / g2);
  }
  rmin[e] = r;
}

// the trial point p = s + step d (rows for t < 3E, variables for t < 3n)
__global__ void k_l1_trial(PdState s, PdDir d, const double* __restrict__ dx, const double* __restrict__ Atdv, uint32_t nr, uint32_t nv,
                           double step, PdState p) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nr) {
    p.Ax[i] = s.Ax[i] + step * d.Adx[i];
    p.u[i] = s.u[i] + step * d.du[i];
    p.l1[i] = s.l1[i] + step * d.dl1[i];
    p.l2[i] = s.l2[i] + step * d.dl2[i];
  }
  if (i < nv) {
    p.x[i] = s.x[i] + step * dx[i];
    p.Atv[i] = s.Atv[i] + step * Atdv[i];
  }
}

// per row of the IRLS step: w = sigma^2 / (b^2 + sigma^2)^2 and w b
__global__ void k_l1_irls(const double* __restrict__ b, uint32_t nr, double s2, double* __restrict__ w, double* __restrict__ wb) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  const double t = b[i] * b[i] + s2;
  const double wi = s2 / (t * t);
  w[i] = wi;
  wb[i] = wi * b[i];
}

// out[0] = sum v (op 0), max |v| (op 1) or min(1, min v) (op 2) over v[0..n), one CTA in a fixed order
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_l1_reduce(int op, const double* __restrict__ v, uint32_t n, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double s = op == 2 ? 1.0 : 0.0;
  for (uint32_t i = threadIdx.x; i < n; i += kThreads) {
    if (op == 0) s += v[i];
    else if (op == 1) s = fmax(s, fabs(v[i]));
    else s = fmin(s, v[i]);
  }
  if (op == 2) {  // block_max_fixed starts from 0, so the minimum has its own tree
    for (int o = 16; o >= 1; o >>= 1) s = fmin(s, __shfl_xor_sync(0xffffffffu, s, o));
    if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 1.0;
    for (int w = 0; w < kThreads / 32; ++w) s = fmin(s, red[w]);
  } else {
    s = op == 0 ? block_sum_fixed<kThreads>(s, red) : block_max_fixed<kThreads>(s, red);
  }
  if (threadIdx.x == 0) out[0] = s;
}

// breadth-first spanning tree from local 0 (R = I), neighbours in ascending order (the incidence lists' order)
std::vector<double> spanning_tree_start(const ra::KeptComponent& K) {
  const uint32_t m = (uint32_t)K.kview.size();
  std::vector<double> R(9 * (size_t)m, 0.0);
  std::vector<char> seen(m, 0);
  std::vector<uint32_t> queue(1, 0);
  R[0] = R[4] = R[8] = 1.0;
  seen[0] = 1;
  for (size_t h = 0; h < queue.size(); ++h) {
    const uint32_t v = queue[h];
    const double* Rv = &R[9 * (size_t)v];
    for (uint32_t p = K.inc_ofs[v]; p < K.inc_ofs[v + 1]; ++p) {
      const uint32_t wv = K.inc_nbr[p], e = K.inc_edge[p];
      if (seen[wv]) continue;
      seen[wv] = 1;
      queue.push_back(wv);
      const double* Q = &K.kR[9 * (size_t)e];
      const bool fwd = K.kab[e].x == v;  // R_w = R_vw R_v, else R_w = R_wv^T R_v
      double* Rw = &R[9 * (size_t)wv];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
          double s = 0.0;
          for (int k = 0; k < 3; ++k) s += (fwd ? Q[3 * i + k] : Q[3 * k + i]) * Rv[3 * k + j];
          Rw[3 * i + j] = s;
        }
    }
  }
  return R;
}

// what r3d_debug_rotavg_l1_step reads back from inside the solver's members (none in rotation_averaging_l1)
struct Trace {
  double* A3 = nullptr;                // 3 (n + 1) n: the systems of each solve as assembled, before they are factored
  std::vector<double> step, resnorm;   // per trial step of the line search: the step and the trial's residual norm
};

// the device side of one call on the kept component
struct Solver {
  r3d_ctx* ctx;
  DeviceWorker& w;
  const uint32_t m, ne, n, nr, nv, P;
  const size_t mstride;
  DevArr<uint32_t> d_iofs, d_inbr, d_iedge;
  DevArr<uint2> d_ab;
  DevArr<double> d_Rk, d_R, d_b, d_cost, d_st[2], d_dir, d_w2, d_sigx, d_rrow, d_dv, d_Atdv, d_rmin, d_part, d_dx, d_A3, d_L, d_Linv,
      d_scal;
  PdState S[2];
  PdDir D;
  int cur = 0;
  // 0 not-positive-definite flag, 1 max|b|, 2 min step ratio, 3 residual norm^2, 4 sum fu^T lambda, 5 max|x|, 6 cost
  double h[8] = {};
  Trace* tr = nullptr;

  Solver(r3d_ctx* c, DeviceWorker& wk, const ra::KeptComponent& K)
      : ctx(c), w(wk), m((uint32_t)K.kview.size()), ne((uint32_t)K.kab.size()), n(m - 1), nr(3 * ne), nv(3 * (m - 1)),
        P(std::max(ne, m - 1)), mstride((size_t)(n + 1) * n), d_iofs(wk), d_inbr(wk), d_iedge(wk), d_ab(wk), d_Rk(wk), d_R(wk), d_b(wk),
        d_cost(wk), d_st{DevArr<double>(wk), DevArr<double>(wk)}, d_dir(wk), d_w2(wk), d_sigx(wk), d_rrow(wk), d_dv(wk), d_Atdv(wk),
        d_rmin(wk), d_part(wk), d_dx(wk), d_A3(wk), d_L(wk), d_Linv(wk), d_scal(wk) {}

  cudaError_t h2d(void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, w.stream); }

  int init(const ra::KeptComponent& K, const std::vector<double>& R0) {
    const int nblk = ((int)n + kCholNB - 1) / kCholNB;
    const size_t st = 4 * (size_t)nr + 2 * (size_t)nv;
    if (!d_iofs.alloc(m + 1) || !d_inbr.alloc(2 * (size_t)ne) || !d_iedge.alloc(2 * (size_t)ne) || !d_ab.alloc(ne) || !d_Rk.alloc(9 * (size_t)ne) ||
        !d_R.alloc(9 * (size_t)m) || !d_b.alloc(nr) || !d_cost.alloc(ne) || !d_st[0].alloc(st) || !d_st[1].alloc(st) ||
        !d_dir.alloc(4 * (size_t)nr) || !d_w2.alloc(nr) || !d_sigx.alloc(nr) || !d_rrow.alloc(nr) || !d_dv.alloc(nr) || !d_Atdv.alloc(nv) ||
        !d_rmin.alloc(ne) || !d_part.alloc(2 * (size_t)P) || !d_dx.alloc(nv) || !d_A3.alloc(3 * mstride) || !d_L.alloc(mstride + 64) ||
        !d_Linv.alloc((size_t)nblk * kCholNB * kCholNB) || !d_scal.alloc(8))
      return fail(ctx, R3D_ERR_NOMEM, "r3d_rotation_averaging_l1: device scratch");
    for (int q = 0; q < 2; ++q) {
      double* p = d_st[q].p;
      S[q] = PdState{p, p + nv, p + nv + nr, p + nv + 2 * (size_t)nr, p + nv + 3 * (size_t)nr, p + nv + 4 * (size_t)nr};
    }
    double* p = d_dir.p;
    D = PdDir{p, p + nr, p + 2 * (size_t)nr, p + 3 * (size_t)nr};
    R3D_CUDA_TRY(ctx, h2d(d_iofs.p, K.inc_ofs.data(), (m + 1) * sizeof(uint32_t)));
    R3D_CUDA_TRY(ctx, h2d(d_inbr.p, K.inc_nbr.data(), K.inc_nbr.size() * sizeof(uint32_t)));
    R3D_CUDA_TRY(ctx, h2d(d_iedge.p, K.inc_edge.data(), K.inc_edge.size() * sizeof(uint32_t)));
    R3D_CUDA_TRY(ctx, h2d(d_ab.p, K.kab.data(), ne * sizeof(uint2)));
    R3D_CUDA_TRY(ctx, h2d(d_Rk.p, K.kR.data(), K.kR.size() * sizeof(double)));
    R3D_CUDA_TRY(ctx, h2d(d_R.p, R0.data(), R0.size() * sizeof(double)));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_scal.p, 0, 8 * sizeof(double), w.stream));
    return R3D_OK;
  }

  int read() {
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(h, d_scal.p, sizeof(h), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    return R3D_OK;
  }
  void reduce(int op, const double* v, uint32_t len, int slot) {
    k_l1_reduce<kRThreads><<<1, kRThreads, 0, w.stream>>>(op, v, len, d_scal.p + slot);
  }
  static uint32_t blocks(uint32_t t) { return (t + 127) / 128; }

  // the residuals b at the current rotations, max |b| into h[1] and the L1 cost into h[6]
  int residuals() {
    k_l1_residual<<<blocks(ne), 128, 0, w.stream>>>(d_R.p, d_ab.p, d_Rk.p, ne, d_b.p, d_cost.p);
    reduce(1, d_b.p, nr, 1);
    reduce(0, d_cost.p, ne, 6);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return read();
  }

  // (A^T diag(wt) A) dx = A^T v, three Laplacians factored one after the other; *not_pd when one is not positive definite
  int solve(const double* wt, const double* v, bool* not_pd) {
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_A3.p, 0, 3 * mstride * sizeof(double), w.stream));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_scal.p, 0, sizeof(double), w.stream));
    k_l1_system<<<n, 128, 0, w.stream>>>(d_iofs.p, d_inbr.p, d_iedge.p, d_ab.p, wt, v, n, mstride, d_A3.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if (tr && tr->A3)
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(tr->A3, d_A3.p, 3 * mstride * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
    int rc;
    for (int k = 0; k < 3; ++k)
      if ((rc = dense_cholesky(ctx, w, d_A3.p + k * mstride, d_L.p, d_Linv.p, (int)n, d_scal.p, d_dx.p + (size_t)k * n))) return rc;
    if ((rc = read())) return rc;
    *not_pd = h[0] != 0.0;
    return R3D_OK;
  }

  // residual norm and duality gap of state q with 1 / tau = tinv into h[3], h[4]
  int norms(int q, double tinv) {
    k_l1_norms<<<blocks(P), 128, 0, w.stream>>>(d_b.p, S[q], ne, n, tinv, P, d_part.p);
    reduce(0, d_part.p, P, 3);
    reduce(0, d_part.p + P, P, 4);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return read();
  }

  // l1decode_pd's start on the residuals in d_b (max |b| in h[1]): S[cur].x = 0, then, unless b = 0 (*zero: x = 0 is
  // the solution), k_l1_pd_start's point in S[cur] with its surrogate duality gap sdg, tau and residual norm
  int pd_start(bool* zero, double& sdg, double& tau, double& resnorm) {
    PdState& s0 = S[cur];
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(s0.x, 0, nv * sizeof(double), w.stream));
    *zero = h[1] == 0.0;
    if (*zero) return R3D_OK;
    k_l1_pd_start<<<blocks(nr), 128, 0, w.stream>>>(d_b.p, d_scal.p + 1, nr, s0, d_dv.p);
    k_l1_at<<<blocks(nv), 128, 0, w.stream>>>(d_iofs.p, d_iedge.p, d_ab.p, d_dv.p, n, s0.Atv);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    int rc;
    if ((rc = norms(cur, 0.0))) return rc;
    sdg = -h[4];
    tau = kPdMu * (2.0 * (double)nr) / sdg;
    if ((rc = norms(cur, 1.0 / tau))) return rc;
    resnorm = std::sqrt(h[3]);
    return R3D_OK;
  }

  // One Newton iteration of l1decode_pd from S[cur] at tau, whose residual norm there is resnorm: the Newton system,
  // the direction, the ratio test (min step ratio in h[2]) and the backtracking line search.  Accepted: S[cur] becomes
  // the trial point and sdg, tau, resnorm its values; else *stuck and S[cur] is unchanged.  *not_pd: the Newton system
  // was not positive definite (nothing after the solve ran).
  int pd_iteration(double& sdg, double& tau, double& resnorm, uint32_t* backtracks, bool* not_pd, bool* stuck) {
    *stuck = false;
    const double tinv = 1.0 / tau;
    const PdState& s = S[cur];
    k_l1_newton<<<blocks(nr), 128, 0, w.stream>>>(d_b.p, s, nr, tinv, d_sigx.p, d_rrow.p, d_w2.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    int rc;
    if ((rc = solve(d_sigx.p, d_rrow.p, not_pd))) return rc;
    if (*not_pd) return R3D_OK;
    k_l1_direction<<<blocks(ne), 128, 0, w.stream>>>(d_ab.p, d_b.p, s, d_w2.p, d_dx.p, ne, n, tinv, D, d_dv.p, d_rmin.p);
    k_l1_at<<<blocks(nv), 128, 0, w.stream>>>(d_iofs.p, d_iedge.p, d_ab.p, d_dv.p, n, d_Atdv.p);
    reduce(2, d_rmin.p, ne, 2);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if ((rc = read())) return rc;
    double step = 0.99 * h[2];
    bool ok = false;
    for (int bt = 0; bt <= kPdMaxBacktracks; ++bt) {
      k_l1_trial<<<blocks(std::max(nr, nv)), 128, 0, w.stream>>>(s, D, d_dx.p, d_Atdv.p, nr, nv, step, S[1 - cur]);
      R3D_CUDA_TRY(ctx, cudaGetLastError());
      if ((rc = norms(1 - cur, tinv))) return rc;
      if (tr) {
        tr->step.push_back(step);
        tr->resnorm.push_back(std::sqrt(h[3]));
      }
      if (std::sqrt(h[3]) <= (1.0 - kPdAlpha * step) * resnorm) {
        ok = true;
        break;
      }
      ++*backtracks;
      step = kPdBeta * step;
    }
    if (!ok) {
      *stuck = true;
      return R3D_OK;
    }
    cur = 1 - cur;
    sdg = -h[4];
    tau = kPdMu * (2.0 * (double)nr) / sdg;
    if ((rc = norms(cur, 1.0 / tau))) return rc;
    resnorm = std::sqrt(h[3]);
    return R3D_OK;
  }

  // l1decode_pd on the residuals in d_b (max |b| in h[1]); the solution is S[cur].x.  *not_pd: a Newton system was not
  // positive definite.
  int l1_regression(uint32_t* iters, uint32_t* backtracks, bool* not_pd) {
    *not_pd = false;
    bool zero = false, stuck = false;
    double sdg = 0.0, tau = 0.0, resnorm = 0.0;
    int rc;
    if ((rc = pd_start(&zero, sdg, tau, resnorm))) return rc;
    if (zero) return R3D_OK;
    for (int it = 0; !(sdg < kPdTol || it >= kPdMaxIter);) {
      ++it;
      ++*iters;
      if ((rc = pd_iteration(sdg, tau, resnorm, backtracks, not_pd, &stuck))) return rc;
      if (*not_pd || stuck) break;  // stuck: the last iterate
    }
    return R3D_OK;
  }

  // One IRLS iteration at the current rotations: the residuals, the Geman-McClure weights w (d_sigx) and w b (d_rrow)
  // with s2 = sigma^2, the weighted normal equations and R <- R exp(dx) (max |dx| in h[5]).  *not_pd: the system was not
  // positive definite (nothing after the solve ran).
  int irls_iteration(double s2, bool* not_pd) {
    int rc;
    if ((rc = residuals())) return rc;
    k_l1_irls<<<blocks(nr), 128, 0, w.stream>>>(d_b.p, nr, s2, d_sigx.p, d_rrow.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if ((rc = solve(d_sigx.p, d_rrow.p, not_pd))) return rc;
    if (*not_pd) return R3D_OK;
    return rotate(d_dx.p);
  }
  static double irls_s2(const r3d_rotavg_l1_options& opt) {
    const double sg = opt.irls_sigma_deg * (R3D_PI / 180.0);
    return sg * sg;
  }

  // R <- R exp(x) with x = the current solution; max |x| into h[5]
  int rotate(const double* x) {
    k_l1_rotate<<<blocks(n), 128, 0, w.stream>>>(x, n, d_R.p);
    reduce(1, x, nv, 5);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    return read();
  }
};

int rotation_averaging_l1(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views, const r3d_rotavg_l1_options& opt,
                          double* rotations, uint8_t* view_kept, uint8_t* edge_kept, uint32_t* edge_support, r3d_rotavg_l1_summary& S) {
  const double t0 = now_ms();
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::memset(rotations, 0, (size_t)n_views * 9 * sizeof(double));
  ra::KeptComponent K;
  int rc = ra::select_component(ctx, "r3d_rotation_averaging_l1: ", rel, n_rel, n_views, opt.max_angular_error_deg, view_kept, edge_kept,
                                edge_support, K);
  S.n_edges = K.n_edges;
  S.n_triplets = K.n_triplets;
  S.n_valid_triplets = K.n_valid_triplets;
  S.ms_triplets = K.ms_triplets;
  if (rc) return rc;
  if (K.kview.empty()) {
    S.ms_device_total = S.ms_triplets;
    S.ms_host = now_ms() - t0 - S.ms_device_total;
    return R3D_OK;
  }
  const uint32_t m = (uint32_t)K.kview.size();
  S.success = 1;
  S.n_kept_views = m;
  S.n_kept_edges = K.kab.size();
  // ---- the spanning-tree start ----
  const double ti = now_ms();
  std::vector<double> R0 = spanning_tree_start(K);
  S.ms_init = now_ms() - ti;
  Solver L(ctx, w, K);
  if ((rc = L.init(K, R0))) return rc;
  Events<3> ev;
  R3D_CUDA_TRY(ctx, ev.create());
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[0], w.stream));
  if ((rc = L.residuals())) return rc;
  S.initial_l1_cost = L.h[6];
  // ---- L1RA ----
  int term = 1;
  bool not_pd = false;
  for (int it = 0; it < opt.l1_max_iterations; ++it) {
    if (it > 0 && (rc = L.residuals())) return rc;
    if ((rc = L.l1_regression(&S.pd_iterations, &S.pd_backtracks, &not_pd))) return rc;
    if (not_pd) {
      term = 2;
      break;
    }
    if ((rc = L.rotate(L.S[L.cur].x))) return rc;
    ++S.l1_iterations;
    if (L.h[5] <= opt.tolerance) {
      term = 0;
      break;
    }
  }
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[1], w.stream));
  // ---- IRLS ----
  if (term != 2 && opt.irls_max_iterations > 0) {
    term = 1;
    const double s2 = Solver::irls_s2(opt);
    for (int it = 0; it < opt.irls_max_iterations; ++it) {
      if ((rc = L.irls_iteration(s2, &not_pd))) return rc;
      if (not_pd) {
        term = 2;
        break;
      }
      ++S.irls_iterations;
      if (L.h[5] <= opt.tolerance) {
        term = 0;
        break;
      }
    }
  }
  if ((rc = L.residuals())) return rc;
  S.final_l1_cost = L.h[6];
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[2], w.stream));
  std::vector<double> R(9 * (size_t)m);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(R.data(), L.d_R.p, R.size() * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  S.termination = term;
  S.ms_l1 = ev.ms(0, 1);
  S.ms_irls = ev.ms(1, 2);
  // the gauge: local 0 is never updated and holds R = I exactly, so R_v R_0^T = R_v
  for (uint32_t a = 0; a < m; ++a) std::memcpy(rotations + 9 * (size_t)K.kview[a], &R[9 * (size_t)a], 9 * sizeof(double));
  S.ms_device_total = S.ms_triplets + S.ms_l1 + S.ms_irls;
  S.ms_host = now_ms() - t0 - S.ms_device_total;
  return R3D_OK;
}

// r3d_debug_rotavg_l1_step: one step of the members above on the kept component
int debug_step(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views, const r3d_rotavg_l1_options& opt,
               const double* rotations, int kind, const double* state, uint64_t n_state, double tau_in, const double* weights,
               const double* rhs, uint32_t n_systems, r3d_rotavg_l1_step_out& O) {
  const char* fn = "r3d_debug_rotavg_l1_step: ";
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::vector<uint8_t> vk(std::max(n_views, 1u));
  ra::KeptComponent K;
  int rc = ra::select_component(ctx, fn, rel, n_rel, n_views, opt.max_angular_error_deg, vk.data(), nullptr, nullptr, K);
  if (rc) return rc;
  if (K.kview.empty()) return R3D_OK;
  const uint32_t m = (uint32_t)K.kview.size(), ne = (uint32_t)K.kab.size(), n = m - 1;
  const size_t nr = 3 * (size_t)ne, nv = 3 * (size_t)n, nst = 4 * nr + 2 * nv;
  if (kind == 0 && state && n_state != nst) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "the state must hold 12 E + 6 n values");
  if (kind == 0 && state && !(std::isfinite(tau_in) && tau_in > 0.0)) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "tau <= 0");
  std::vector<double> R0;
  if (!rotations) {
    R0 = spanning_tree_start(K);
  } else {
    R0.resize(9 * (size_t)m);
    for (uint32_t a = 0; a < m; ++a) std::memcpy(&R0[9 * (size_t)a], rotations + 9 * (size_t)K.kview[a], 9 * sizeof(double));
    for (double v : R0)
      if (!std::isfinite(v)) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "non-finite rotations");
  }
  O.n_kept_views = m;
  O.n_kept_edges = ne;
  for (uint32_t a = 0; a < m; ++a)
    if (O.view_ids) O.view_ids[a] = K.kview[a];
  for (uint32_t e = 0; e < ne; ++e)
    if (O.ab) {
      O.ab[2 * (size_t)e] = K.kab[e].x;
      O.ab[2 * (size_t)e + 1] = K.kab[e].y;
    }
  if (O.Rk) std::memcpy(O.Rk, K.kR.data(), K.kR.size() * sizeof(double));
  if (O.rotations0) std::memcpy(O.rotations0, R0.data(), R0.size() * sizeof(double));
  Solver L(ctx, w, K);
  if ((rc = L.init(K, R0))) return rc;
  Trace T;
  auto d2h = [&](void* dst, const void* src, size_t bytes) -> int {
    if (dst) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, w.stream));
    return R3D_OK;
  };
  auto sync = [&]() -> int {
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    return R3D_OK;
  };
  auto residual_out = [&]() -> int {
    O.bmax = L.h[1];
    if ((rc = d2h(O.b, L.d_b.p, nr * sizeof(double))) || (rc = d2h(O.cost, L.d_cost.p, ne * sizeof(double)))) return rc;
    return sync();
  };
  auto rotations_out = [&]() -> int {
    O.xmax = L.h[5];
    if ((rc = d2h(O.rotations, L.d_R.p, 9 * (size_t)m * sizeof(double)))) return rc;
    return sync();
  };
  const size_t lap = 3 * L.mstride;
  if (kind == 1) {
    T.A3 = O.laplacians;
    L.tr = &T;
    bool not_pd = false;
    if ((rc = L.irls_iteration(Solver::irls_s2(opt), &not_pd)) || (rc = residual_out())) return rc;
    O.not_pd = not_pd;
    if ((rc = d2h(O.w, L.d_sigx.p, nr * sizeof(double))) || (rc = d2h(O.wb, L.d_rrow.p, nr * sizeof(double)))) return rc;
    if (not_pd) return sync();
    if ((rc = d2h(O.dx, L.d_dx.p, nv * sizeof(double)))) return rc;
    return rotations_out();
  }
  if ((rc = L.residuals()) || (rc = residual_out())) return rc;
  if (kind == 2) {
    for (uint32_t q = 0; q < n_systems; ++q) {
      T.A3 = O.laplacians ? O.laplacians + q * lap : nullptr;
      L.tr = &T;
      R3D_CUDA_TRY(ctx, L.h2d(L.d_sigx.p, weights + q * nr, nr * sizeof(double)));
      R3D_CUDA_TRY(ctx, L.h2d(L.d_rrow.p, rhs + q * nr, nr * sizeof(double)));
      bool not_pd = false;
      if ((rc = L.solve(L.d_sigx.p, L.d_rrow.p, &not_pd))) return rc;
      if (O.sys_not_pd) O.sys_not_pd[q] = not_pd;
      if (!not_pd && O.dx && (rc = d2h(O.dx + q * nv, L.d_dx.p, nv * sizeof(double)))) return rc;
    }
    return sync();
  }
  // kind 0
  double sdg = 0.0, tau = 0.0, resnorm = 0.0;
  if (!state) {
    bool zero = false;
    if ((rc = L.pd_start(&zero, sdg, tau, resnorm))) return rc;
    if (zero) {
      O.b_zero = 1;
      if ((rc = L.rotate(L.S[L.cur].x))) return rc;
      return rotations_out();
    }
  } else {
    std::vector<double> bh(nr);
    if ((rc = d2h(bh.data(), L.d_b.p, nr * sizeof(double))) || (rc = sync())) return rc;
    for (size_t i = 0; i < nst; ++i)
      if (!std::isfinite(state[i])) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "a non-finite state");
    const double *Ax = state + nv, *u = Ax + nr, *l1 = u + nr, *l2 = l1 + nr;
    for (size_t i = 0; i < nr; ++i) {
      const double f1 = (Ax[i] - bh[i]) - u[i], f2 = (-Ax[i] + bh[i]) - u[i];
      if (!(f1 < 0.0) || !(f2 < 0.0) || !(l1[i] > 0.0) || !(l2[i] > 0.0))
        return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "u or lambda outside the interior");
    }
    R3D_CUDA_TRY(ctx, L.h2d(L.d_st[L.cur].p, state, nst * sizeof(double)));
    tau = tau_in;
    if ((rc = L.norms(L.cur, 1.0 / tau))) return rc;
    sdg = -L.h[4];
    resnorm = std::sqrt(L.h[3]);
  }
  O.sdg0 = sdg;
  O.tau0 = tau;
  O.resnorm0 = resnorm;
  if ((rc = d2h(O.state0, L.d_st[L.cur].p, nst * sizeof(double)))) return rc;
  T.A3 = O.laplacians;
  L.tr = &T;
  uint32_t backtracks = 0;
  bool not_pd = false, stuck = false;
  if ((rc = L.pd_iteration(sdg, tau, resnorm, &backtracks, &not_pd, &stuck))) return rc;
  O.not_pd = not_pd;
  if ((rc = d2h(O.sigx, L.d_sigx.p, nr * sizeof(double))) || (rc = d2h(O.rrow, L.d_rrow.p, nr * sizeof(double))) ||
      (rc = d2h(O.w2, L.d_w2.p, nr * sizeof(double))))
    return rc;
  if (not_pd) return sync();
  O.step_max = L.h[2];
  O.n_trials = (uint32_t)T.step.size();
  for (uint32_t t = 0; t < O.n_trials; ++t) {
    O.trial_step[t] = T.step[t];
    O.trial_resnorm[t] = T.resnorm[t];
  }
  O.accepted = !stuck;
  O.sdg = sdg;
  O.tau = tau;
  O.resnorm = resnorm;
  if ((rc = d2h(O.dx, L.d_dx.p, nv * sizeof(double))) || (rc = d2h(O.Adx, L.D.Adx, nr * sizeof(double))) ||
      (rc = d2h(O.du, L.D.du, nr * sizeof(double))) || (rc = d2h(O.dl1, L.D.dl1, nr * sizeof(double))) ||
      (rc = d2h(O.dl2, L.D.dl2, nr * sizeof(double))) || (rc = d2h(O.Atdv, L.d_Atdv.p, nv * sizeof(double))) ||
      (rc = d2h(O.rmin, L.d_rmin.p, ne * sizeof(double))) || (rc = d2h(O.state, L.d_st[L.cur].p, nst * sizeof(double))))
    return rc;
  if ((rc = L.rotate(L.S[L.cur].x))) return rc;
  return rotations_out();
}

}  // namespace rl
}  // namespace r3d

using namespace r3d;

extern "C" void r3d_rotavg_l1_default_options(r3d_rotavg_l1_options* o) {
  if (!o) return;
  o->max_angular_error_deg = 5.0;
  o->irls_sigma_deg = 5.0;
  o->l1_max_iterations = 32;
  o->irls_max_iterations = 32;
  o->tolerance = 1e-5;
}

extern "C" int r3d_rotation_averaging_l1(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                                         const r3d_rotavg_l1_options* opt, double* rotations, uint8_t* view_kept, uint8_t* edge_kept,
                                         uint32_t* edge_support, r3d_rotavg_l1_summary* summary) {
  if (!ctx || (!rel && n_rel) || !opt || (!rotations && n_views) || (!view_kept && n_views) || !summary)
    return fail(ctx, R3D_ERR_INVALID, "r3d_rotation_averaging_l1: bad arguments");
  std::memset(summary, 0, sizeof(*summary));
  summary->termination = -1;
  if (!(opt->max_angular_error_deg > 0.0)) return fail(ctx, R3D_ERR_INVALID, "r3d_rotation_averaging_l1: max_angular_error_deg <= 0");
  if (opt->l1_max_iterations < 1 || opt->irls_max_iterations < 0 || !(opt->tolerance > 0.0) || !(opt->irls_sigma_deg > 0.0))
    return fail(ctx, R3D_ERR_INVALID, "r3d_rotation_averaging_l1: an iteration cap below its minimum, or tolerance / sigma <= 0");
  return rl::rotation_averaging_l1(ctx, rel, n_rel, n_views, *opt, rotations, view_kept, edge_kept, edge_support, *summary);
}

extern "C" int r3d_debug_rotavg_l1_step(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                                        const r3d_rotavg_l1_options* opt, const double* rotations, int kind, const double* state,
                                        uint64_t n_state, double tau, const double* weights, const double* rhs, uint32_t n_systems,
                                        r3d_rotavg_l1_step_out* out) {
  static_assert(sizeof(out->trial_step) / sizeof(double) == rl::kPdMaxBacktracks + 1, "one slot per trial step");
  if (!ctx || (!rel && n_rel) || !opt || kind < 0 || kind > 2 || (!state && n_state) || (kind != 0 && state) ||
      (kind == 2 && (!weights || !rhs || n_systems < 1)) || !out)
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_rotavg_l1_step: bad arguments");
  if (!(opt->max_angular_error_deg > 0.0) || !(opt->irls_sigma_deg > 0.0))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_rotavg_l1_step: max_angular_error_deg or irls_sigma_deg <= 0");
  r3d_rotavg_l1_step_out& O = *out;
  O.n_kept_views = O.n_kept_edges = 0;
  O.bmax = O.sdg0 = O.tau0 = O.resnorm0 = O.step_max = O.sdg = O.tau = O.resnorm = O.xmax = 0.0;
  O.b_zero = O.not_pd = O.accepted = 0;
  O.n_trials = 0;
  std::memset(O.trial_step, 0, sizeof(O.trial_step));
  std::memset(O.trial_resnorm, 0, sizeof(O.trial_resnorm));
  return rl::debug_step(ctx, rel, n_rel, n_views, *opt, rotations, kind, state, n_state, tau, weights, rhs, n_systems, O);
}
