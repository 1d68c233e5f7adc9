// rotavg.cu -- global camera rotations from the relative motions (r3d_rotation_averaging), and the largest
// bi-edge-connected component of a match graph (r3d_matches_keep_largest_biedge_component, host only).
// COMPILED WITH --fmad=false (regard3d_b200/build.py): the triplet decisions must equal the CPU restatement's
// (oracle/oracle_rotavg.cpp) bit for bit, so the cycle trace is written out in one fixed product order on both sides and
// the angle goes through detmath.cuh's acos.
//
// Replaces GlobalSfM_Rotation_AveragingSolver::Run with ROTATION_AVERAGING_L2 (OpenMVG 1.4, SURVEY.md A.10):
//   1. k_rotavg_triplets: every triangle {i < j < k} of the edge graph, from an upper-adjacency CSR (neighbours > self,
//      sorted; edge id = CSR position).  One CTA per node i (dynamic work counter): up(i) is scattered into a shared
//      node -> edge table, then one warp per edge (i, j) walks up(j) and looks each k up in the table.  Per triangle
//      the cycle trace of R_ik^T R_jk R_ij, a two-tier decision (cos bounds away from the threshold, the exact
//      float(acos) test inside the band) and integer atomics on the support of its three edges.
//   2. host: bridges (Tarjan) and the largest 2-edge-connected component of the supported edges, reindexing.
//      Steps 1 and 2 are select_component, which the L1 method (rotavg_l1.cu) shares.
//   3. L2 initialisation: M = A^T A assembled by one owner per block row, M + sigma I factored once by k_chol_fused
//      (ba.cu), block inverse iteration with 3 right-hand sides (k_rotavg_trsm3: blocked forward / backward
//      substitution, one cooperative launch) and a 3 x 3 Cholesky-QR (k_rotavg_orth), then the sign, the SO(3)
//      projection of every 3 x 3 block (relpose_math.cuh's Jacobi SVD) and the gauge (k_rotavg_project).
//   4. refinement: Levenberg-Marquardt (averaging.cuh's loop around lm_trust_region.cuh's trust region) on the
//      angle-axis of every kept view: k_rotavg_eval (residual log(R_ij^T R_j R_i^T) with forward-mode duals),
//      k_rotavg_system (dense normal equations by one owner per block row, no floating-point atomics), k_chol_fused,
//      fixed-order reductions: repeated calls are bit-identical.
#include "r3d_internal.cuh"
#include "averaging.cuh"
#include "ba_model.cuh"
#include "detmath.cuh"
#include "relpose_math.cuh"

#include <cooperative_groups.h>

#include <cmath>
#include <cstring>
#include <numeric>

namespace cg = cooperative_groups;

namespace r3d {
namespace ra {

constexpr uint32_t kMaxTripletNodes = 57344;  // node -> edge table of one CTA in shared memory (224 KB)
constexpr double kSigmaRel = 1e-7;            // shift of the inverse iteration: sigma = kSigmaRel * max degree
constexpr double kInitTol = 1e-12;            // stop when || Q_new - Q_old (Q_old^T Q_new) ||_F < kInitTol
constexpr uint32_t kInitMaxIter = 100;
constexpr double kCycleBand = 1e-6;           // cos band around the threshold inside which the exact test runs

// ---- 1. triplets ------------------------------------------------------------------------------------------------
// The decision both sides take: float(R2D(acos(clamp((trace - 1) / 2, -1, 1)))) < thr
R3D_RP_HD double cycle_trace(const double* Rij, const double* Rjk, const double* Rik) {
  double tr = 0.0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      const double t = Rjk[3 * a] * Rij[b] + Rjk[3 * a + 1] * Rij[3 + b] + Rjk[3 * a + 2] * Rij[6 + b];  // (R_jk R_ij)[a][b]
      tr = tr + Rik[3 * a + b] * t;                                                                     // trace(R_ik^T T)
    }
  return tr;
}
R3D_RP_HD double cycle_cos(double tr) {
  double c = (tr - 1.0) / 2.0;
  if (c > 1.0) c = 1.0;
  if (c < -1.0) c = -1.0;
  return c;
}
R3D_RP_HD bool cycle_valid_exact(double c, float thr) {
  const double deg = dm::acos_det(c) / R3D_PI * 180.0;  // R2D
  return (float)deg < thr;
}

constexpr int kTThreads = 256;
constexpr int kTWarps = kTThreads / 32;

__global__ void __launch_bounds__(kTThreads) k_rotavg_triplets(const uint32_t* __restrict__ up_ofs, const uint32_t* __restrict__ up_nbr,
                                                               uint32_t n_nodes, const double* __restrict__ rot, uint32_t E, double c_lo,
                                                               double c_hi, float thr, uint32_t* __restrict__ work,
                                                               uint32_t* __restrict__ support, unsigned long long* __restrict__ counts) {
  extern __shared__ int32_t slot[];  // node k -> CSR position of (i, k), -1 if k is not in up(i)
  __shared__ uint32_t s_node;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  for (uint32_t k = tid; k < n_nodes; k += kTThreads) slot[k] = -1;
  unsigned long long nt = 0, nv = 0;
  for (;;) {
    __syncthreads();
    if (tid == 0) s_node = atomicAdd(work, 1u);
    __syncthreads();
    const uint32_t i = s_node;
    if (i >= n_nodes) break;
    const uint32_t b = up_ofs[i], e = up_ofs[i + 1];
    for (uint32_t p = b + tid; p < e; p += kTThreads) slot[up_nbr[p]] = (int32_t)p;
    __syncthreads();
    for (uint32_t p = b + warp; p < e; p += kTWarps) {
      const uint32_t j = up_nbr[p];
      double Rij[9];
      for (int c = 0; c < 9; ++c) Rij[c] = rot[(size_t)c * E + p];
      uint32_t own = 0;
      for (uint32_t q = up_ofs[j] + lane; q < up_ofs[j + 1]; q += 32) {
        const int32_t s = slot[up_nbr[q]];
        if (s < 0) continue;
        double Rjk[9], Rik[9];
        for (int c = 0; c < 9; ++c) {
          Rjk[c] = rot[(size_t)c * E + q];
          Rik[c] = rot[(size_t)c * E + (uint32_t)s];
        }
        const double cs = cycle_cos(cycle_trace(Rij, Rjk, Rik));
        // tier 1: well inside / outside the threshold (cos is monotone, the band is far wider than acos' error and a
        // float ulp); tier 2: the exact test
        const bool ok = cs >= c_hi ? true : (cs <= c_lo ? false : cycle_valid_exact(cs, thr));
        ++nt;
        if (ok) {
          ++nv;
          ++own;
          atomicAdd(&support[q], 1u);
          atomicAdd(&support[s], 1u);
        }
      }
      for (int o = 16; o >= 1; o >>= 1) own += __shfl_xor_sync(0xffffffffu, own, o);
      if (lane == 0 && own) atomicAdd(&support[p], own);
    }
    __syncthreads();
    for (uint32_t p = b + tid; p < e; p += kTThreads) slot[up_nbr[p]] = -1;
  }
  for (int o = 16; o >= 1; o >>= 1) {
    nt += __shfl_xor_sync(0xffffffffu, nt, o);
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
  }
  if (lane == 0) {
    if (nt) atomicAdd(&counts[0], nt);
    if (nv) atomicAdd(&counts[1], nv);
  }
}

// ---- 3. L2 initialisation ---------------------------------------------------------------------------------------
// One thread per (view a, incident edge): the block (a, b) of M = A^T A, A = one block row [R_ab | -I] per edge (X_b =
// R_ab X_a): M_ab = -R_ab^T (a < b), M_ab = -R_ba (a > b); one thread per view: the diagonal deg(a) + sigma.  Every
// entry is written once into the zeroed (N + 1) x N matrix (row N: the unused right-hand side of k_chol_fused).
__global__ void k_rotavg_assemble_M(const uint32_t* __restrict__ inc_ofs, const uint32_t* __restrict__ inc_nbr,
                                    const uint32_t* __restrict__ inc_edge, const double* __restrict__ Rk, uint32_t m, double sigma,
                                    double* __restrict__ A) {
  const uint32_t N = 3 * m;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m) {
    const double d = (double)(inc_ofs[t + 1] - inc_ofs[t]) + sigma;
    for (int r = 0; r < 3; ++r) A[(size_t)(3 * t + r) * N + 3 * t + r] = d;
  }
  const uint32_t n_inc = inc_ofs[m];
  if (t >= n_inc) return;
  uint32_t lo = 0, hi = m;  // owner view of incidence entry t
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (inc_ofs[mid] <= t) lo = mid;
    else hi = mid;
  }
  const uint32_t a = lo, b = inc_nbr[t];
  const double* R = Rk + 9 * (size_t)inc_edge[t];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) A[(size_t)(3 * a + r) * N + 3 * b + c] = a < b ? -R[3 * c + r] : -R[3 * r + c];
}

// L Lt Y = Y for 3 right-hand sides (Y: n x 3 row-major), with the factor of k_chol_fused (L row-major n-stride, Linv =
// inverses of its 32 x 32 diagonal blocks).  Blocked and right-looking like k_chol_fused's own substitution: per panel
// every CTA forms y_k = Linv_k b_k itself, then the rows outside the panel are updated strided over the grid (forward:
// one warp per row, a fixed shuffle tree over the panel's 32 columns; backward: one thread per row) and one grid
// barrier orders the panel.  The forward result goes to Z, the solution back to Y, so no CTA reads a row another one
// writes inside the same panel.
constexpr int kSThreads = 256;
__global__ void __launch_bounds__(kSThreads, 1) k_rotavg_trsm3(const double* __restrict__ L, const double* __restrict__ Linv, int n,
                                                            double* __restrict__ Y, double* __restrict__ Z) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double yk[kCholNB * 3];
  const int tid = threadIdx.x, lane = tid & 31;
  const int gw = (int)((blockIdx.x * blockDim.x + tid) >> 5), n_gw = (int)(gridDim.x * blockDim.x / 32);
  const int gt = (int)(blockIdx.x * blockDim.x + tid), n_gt = (int)(gridDim.x * blockDim.x);
  const int nblk = (n + kCholNB - 1) / kCholNB;
  for (int kbi = 0; kbi < nblk; ++kbi) {
    const int k0 = kbi * kCholNB, kb = min(kCholNB, n - k0);
    const double* Li = Linv + (size_t)kbi * kCholNB * kCholNB;
    if (tid < 3 * kCholNB) {
      const int r = tid / 3, c = tid % 3;
      double s = 0.0;
      if (r < kb)
        for (int t = 0; t <= r; ++t) s += Li[r * kCholNB + t] * Y[3 * (size_t)(k0 + t) + c];
      yk[tid] = s;
    }
    __syncthreads();
    if (blockIdx.x == 0 && tid < 3 * kb) Z[3 * (size_t)k0 + tid] = yk[tid];
    for (int i = k0 + kb + gw; i < n; i += n_gw) {
      const double l = lane < kb ? L[(size_t)i * n + k0 + lane] : 0.0;
      double v0 = l * yk[3 * lane], v1 = l * yk[3 * lane + 1], v2 = l * yk[3 * lane + 2];
      for (int o = 16; o >= 1; o >>= 1) {
        v0 += __shfl_xor_sync(0xffffffffu, v0, o);
        v1 += __shfl_xor_sync(0xffffffffu, v1, o);
        v2 += __shfl_xor_sync(0xffffffffu, v2, o);
      }
      if (lane == 0) {
        Y[3 * (size_t)i] -= v0;
        Y[3 * (size_t)i + 1] -= v1;
        Y[3 * (size_t)i + 2] -= v2;
      }
    }
    grid.sync();
  }
  for (int kbi = nblk - 1; kbi >= 0; --kbi) {
    const int k0 = kbi * kCholNB, kb = min(kCholNB, n - k0);
    const double* Li = Linv + (size_t)kbi * kCholNB * kCholNB;
    if (tid < 3 * kCholNB) {  // x_k = Linv_k^T z_k
      const int r = tid / 3, c = tid % 3;
      double s = 0.0;
      if (r < kb)
        for (int t = r; t < kb; ++t) s += Li[t * kCholNB + r] * Z[3 * (size_t)(k0 + t) + c];
      yk[tid] = s;
    }
    __syncthreads();
    if (blockIdx.x == 0 && tid < 3 * kb) Y[3 * (size_t)k0 + tid] = yk[tid];
    for (int j = gt; j < k0; j += n_gt) {
      double s0 = 0.0, s1 = 0.0, s2 = 0.0;
      for (int t = 0; t < kb; ++t) {
        const double l = L[(size_t)(k0 + t) * n + j];
        s0 += l * yk[3 * t];
        s1 += l * yk[3 * t + 1];
        s2 += l * yk[3 * t + 2];
      }
      Z[3 * (size_t)j] -= s0;
      Z[3 * (size_t)j + 1] -= s1;
      Z[3 * (size_t)j + 2] -= s2;
    }
    grid.sync();
  }
}

// Cholesky-QR of Y (n x 3): G = Y^T Y = L3 L3^T, Q_new = Y L3^-T; with first = 0 also C = Q^T Q_new and the subspace
// change || Q_new - Q C ||_F -> out[0].  Q and Y both receive Q_new.  One CTA, fixed-order reductions.
constexpr int kOThreads = 256;
__global__ void __launch_bounds__(kOThreads) k_rotavg_orth(double* __restrict__ Y, double* __restrict__ Q, int n, int first,
                                                           double* __restrict__ out) {
  __shared__ double red[kOThreads / 32];
  __shared__ double Li[9], Cm[9];
  const int tid = threadIdx.x;
  double g[6] = {0, 0, 0, 0, 0, 0};
  for (int i = tid; i < n; i += kOThreads) {
    const double y0 = Y[3 * (size_t)i], y1 = Y[3 * (size_t)i + 1], y2 = Y[3 * (size_t)i + 2];
    g[0] += y0 * y0; g[1] += y1 * y0; g[2] += y1 * y1; g[3] += y2 * y0; g[4] += y2 * y1; g[5] += y2 * y2;
  }
  for (int k = 0; k < 6; ++k) g[k] = block_sum_fixed<kOThreads>(g[k], red);
  if (tid == 0) {  // L3 = chol(G), Li = L3^-1 (lower)
    const double l00 = sqrt(g[0]);
    const double l10 = g[1] / l00, l20 = g[3] / l00;
    const double l11 = sqrt(g[2] - l10 * l10);
    const double l21 = (g[4] - l20 * l10) / l11;
    const double l22 = sqrt(g[5] - l20 * l20 - l21 * l21);
    Li[0] = 1.0 / l00; Li[1] = 0.0; Li[2] = 0.0;
    Li[4] = 1.0 / l11; Li[3] = -l10 * Li[0] / l11; Li[5] = 0.0;
    Li[8] = 1.0 / l22; Li[7] = -l21 * Li[4] / l22; Li[6] = -(l20 * Li[0] + l21 * Li[3]) / l22;
  }
  __syncthreads();
  // q_new[c] = sum_k y[k] Li[c][k]  (row of Y L3^-T)
  auto qnew = [&](int i, double* q) {
    const double y0 = Y[3 * (size_t)i], y1 = Y[3 * (size_t)i + 1], y2 = Y[3 * (size_t)i + 2];
    for (int c = 0; c < 3; ++c) q[c] = y0 * Li[3 * c] + y1 * Li[3 * c + 1] + y2 * Li[3 * c + 2];
  };
  if (!first) {
    double cm[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = tid; i < n; i += kOThreads) {
      double q[3];
      qnew(i, q);
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) cm[3 * a + b] += Q[3 * (size_t)i + a] * q[b];
    }
    for (int k = 0; k < 9; ++k) {
      const double s = block_sum_fixed<kOThreads>(cm[k], red);
      if (tid == 0) Cm[k] = s;
    }
    __syncthreads();
    double ch = 0.0;
    for (int i = tid; i < n; i += kOThreads) {
      double q[3];
      qnew(i, q);
      for (int b = 0; b < 3; ++b) {
        const double d = q[b] - (Q[3 * (size_t)i] * Cm[b] + Q[3 * (size_t)i + 1] * Cm[3 + b] + Q[3 * (size_t)i + 2] * Cm[6 + b]);
        ch += d * d;
      }
    }
    ch = block_sum_fixed<kOThreads>(ch, red);
    if (tid == 0) out[0] = sqrt(ch);
    __syncthreads();
  }
  for (int i = tid; i < n; i += kOThreads) {
    double q[3];
    qnew(i, q);
    for (int c = 0; c < 3; ++c) Q[3 * (size_t)i + c] = q[c];
  }
  __syncthreads();
  for (int i = tid; i < n; i += kOThreads)
    for (int c = 0; c < 3; ++c) Y[3 * (size_t)i + c] = Q[3 * (size_t)i + c];
}

// R_i = the rotation closest to s X_i (X_i = rows 3i..3i+2 of Q, s = sign of sum_i det X_i): u0 v0^T + u1 v1^T +
// (u0 x u1)(v0 x v1)^T from the fixed-sweep Jacobi SVD; then the gauge R_i <- R_i R_0^T, R_0 = I exactly.
R3D_RP_HD void project_so3(const double* X, double* R) {
  double U[9], S[3], V[9];
  rp::svd3(X, U, S, V);  // U's third column is u0 x u1
  V[2] = V[3] * V[7] - V[6] * V[4];
  V[5] = V[6] * V[1] - V[0] * V[7];
  V[8] = V[0] * V[4] - V[3] * V[1];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[3 * r + c] = U[3 * r] * V[3 * c] + U[3 * r + 1] * V[3 * c + 1] + U[3 * r + 2] * V[3 * c + 2];
}
__global__ void __launch_bounds__(kOThreads) k_rotavg_project(const double* __restrict__ Q, uint32_t m, double* __restrict__ Rout) {
  __shared__ double red[kOThreads / 32];
  __shared__ double R0[9];
  const uint32_t tid = threadIdx.x;
  double dsum = 0.0;
  for (uint32_t i = tid; i < m; i += kOThreads) dsum += rp::det3(Q + 9 * (size_t)i);
  dsum = block_sum_fixed<kOThreads>(dsum, red);
  const double sg = dsum < 0.0 ? -1.0 : 1.0;
  if (tid == 0) {
    double X[9];
    for (int k = 0; k < 9; ++k) X[k] = sg * Q[k];
    project_so3(X, R0);
  }
  __syncthreads();
  for (uint32_t i = tid; i < m; i += kOThreads) {
    double X[9], R[9];
    for (int k = 0; k < 9; ++k) X[k] = sg * Q[9 * (size_t)i + k];
    project_so3(X, R);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        Rout[9 * (size_t)i + 3 * r + c] = i == 0 ? (r == c ? 1.0 : 0.0)
                                                 : R[3 * r] * R0[3 * c] + R[3 * r + 1] * R0[3 * c + 1] + R[3 * r + 2] * R0[3 * c + 2];
  }
}

// ---- 4. refinement ----------------------------------------------------------------------------------------------
// r = log(R_ab^T R_b R_a^T)^v
template <class T>
__device__ void edge_residual(const T* aa_a, const T* aa_b, const double* Rab, T* r) {
  T Ra[9], Rb[9], P[9], E[9];
  aa_to_R(aa_a, Ra);
  aa_to_R(aa_b, Rb);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) P[3 * i + j] = Rb[3 * i] * Ra[3 * j] + Rb[3 * i + 1] * Ra[3 * j + 1] + Rb[3 * i + 2] * Ra[3 * j + 2];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[3 * i + j] = Rab[i] * P[j] + Rab[3 + i] * P[3 + j] + Rab[6 + i] * P[6 + j];
  R_to_aa(E, r);
}

// per kept edge: Corrector-scaled residual (3) and Jacobian (3 x 6: first view's angle-axis, then the second's)
__global__ void k_rotavg_eval(const double* __restrict__ aa, const uint2* __restrict__ ab, const double* __restrict__ Rk, uint32_t ne,
                              double huber_a, double* __restrict__ res, double* __restrict__ jac) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  Dual<6> xa[3], xb[3], r[3];
  for (int k = 0; k < 3; ++k) {
    xa[k] = dconst<6>(aa[3 * (size_t)v.x + k]);
    xa[k].v[k] = 1.0;
    xb[k] = dconst<6>(aa[3 * (size_t)v.y + k]);
    xb[k].v[3 + k] = 1.0;
  }
  edge_residual(xa, xb, Rk + 9 * (size_t)e, r);
  double rho1;
  ba::huber_rho(r[0].a * r[0].a + r[1].a * r[1].a + r[2].a * r[2].a, huber_a, &rho1);
  const double sq = ::sqrt(rho1);  // Corrector, rho'' <= 0 branch
  for (int i = 0; i < 3; ++i) {
    res[3 * (size_t)e + i] = r[i].a * sq;
    for (int k = 0; k < 6; ++k) jac[18 * (size_t)e + 6 * i + k] = r[i].v[k] * sq;
  }
}

// per kept edge: 1/2 rho(|r|^2) at the angle-axis aa
__global__ void k_rotavg_cost(const double* __restrict__ aa, const uint2* __restrict__ ab, const double* __restrict__ Rk, uint32_t ne,
                              double huber_a, double* __restrict__ cost) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  double r[3];
  edge_residual(aa + 3 * (size_t)v.x, aa + 3 * (size_t)v.y, Rk + 9 * (size_t)e, r);
  double rho1;
  cost[e] = 0.5 * ba::huber_rho(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], huber_a, &rho1);
}

// Owner per view a (one CTA), its incident edges in neighbour order: its block row of J^T J + D^2 (scaled after the
// block products) into the zeroed (N + 1) x N system and -g into the right-hand-side row N.  Off-diagonal blocks first,
// one per incident edge.
__global__ void __launch_bounds__(128) k_rotavg_system(const uint32_t* __restrict__ inc_ofs, const uint32_t* __restrict__ inc_nbr,
                                                       const uint32_t* __restrict__ inc_edge, const uint2* __restrict__ ab,
                                                       const double* __restrict__ jac, uint32_t m, double* __restrict__ scale,
                                                       double* __restrict__ g, double* __restrict__ diag, double inv_radius,
                                                       double* __restrict__ A) {
  const uint32_t a = blockIdx.x, tid = threadIdx.x;
  const uint32_t N = 3 * m;
  const uint32_t b0 = inc_ofs[a], b1 = inc_ofs[a + 1];
  auto col = [&](uint32_t e, uint32_t v) -> int { return ab[e].x == v ? 0 : 3; };
  for (uint32_t p = b0 + tid; p < b1; p += blockDim.x) {
    const uint32_t e = inc_edge[p], b = inc_nbr[p];
    const int oa = col(e, a), ob = 3 - oa;
    const double* J = jac + 18 * (size_t)e;
#pragma unroll 1  // rolled: 56 registers, 64 unrolled
    for (int k = 0; k < 3; ++k)
      for (int l = 0; l < 3; ++l) {
        const double s = J[oa + k] * J[ob + l] + J[6 + oa + k] * J[6 + ob + l] + J[12 + oa + k] * J[12 + ob + l];
        A[(size_t)(3 * a + k) * N + 3 * b + l] = s * scale[3 * a + k] * scale[3 * b + l];
      }
  }
  if (tid < 9) {  // diagonal block: sum over the incident edges in order, + D^2
    const int k = (int)tid / 3, l = (int)tid % 3;
    double s = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const int oa = col(e, a);
      const double* J = jac + 18 * (size_t)e;
      s += (J[oa + k] * J[oa + l] + J[6 + oa + k] * J[6 + oa + l]) + J[12 + oa + k] * J[12 + oa + l];
    }
    s = s * scale[3 * a + k] * scale[3 * a + l];
    if (k == l) s += fmin(fmax(diag[3 * a + k], 1e-6), 1e32) * inv_radius;
    A[(size_t)(3 * a + k) * N + 3 * a + l] = s;
    if (tid < 3) A[(size_t)N * N + 3 * a + tid] = -g[3 * a + tid];
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------
// cooperative grid of k_rotavg_trsm3: grid 0 = up to 4 CTAs per SM as occupancy allows (what the inverse iteration
// runs), otherwise the caller's, R3D_ERR_INVALID when that many CTAs cannot be co-resident
int trsm3_grid(r3d_ctx* ctx, DeviceWorker& w, int* grid) {
  int per_sm = 0;
  R3D_CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rotavg_trsm3, kSThreads, 0));
  if (*grid == 0) *grid = w.sm_count * std::max(1, std::min(per_sm, 4));
  if (*grid < 1 || *grid > std::max(per_sm, 0) * w.sm_count)
    return fail(ctx, R3D_ERR_INVALID, "k_rotavg_trsm3: " + std::to_string(*grid) + " CTAs cannot be co-resident");
  return R3D_OK;
}

// L Lt X = Y in place of Y (n x 3), Z: n x 3 scratch; L, Linv from dense_cholesky; grid from trsm3_grid
int trsm3(r3d_ctx* ctx, DeviceWorker& w, const double* L, const double* Linv, int n, double* Y, double* Z, int grid) {
  void* args[] = {&L, &Linv, &n, &Y, &Z};
  R3D_CUDA_TRY(ctx, cudaLaunchCooperativeKernel((void*)k_rotavg_trsm3, dim3(grid), dim3(kSThreads), args, 0, w.stream));
  return R3D_OK;
}

int largest_biedge_component(uint32_t n, const std::vector<uint32_t>& eu, const std::vector<uint32_t>& ev, std::vector<int>& comp) {
  const size_t E = eu.size();
  std::vector<uint32_t> ofs(n + 1, 0);
  for (size_t k = 0; k < E; ++k)
    if (eu[k] != ev[k]) { ofs[eu[k] + 1]++; ofs[ev[k] + 1]++; }
  for (uint32_t v = 0; v < n; ++v) ofs[v + 1] += ofs[v];
  std::vector<std::pair<uint32_t, uint32_t>> adj(ofs[n]);  // (neighbour, edge)
  {
    std::vector<uint32_t> pos(ofs.begin(), ofs.end() - 1);
    for (size_t k = 0; k < E; ++k)
      if (eu[k] != ev[k]) {
        adj[pos[eu[k]]++] = {ev[k], (uint32_t)k};
        adj[pos[ev[k]]++] = {eu[k], (uint32_t)k};
      }
  }
  std::vector<int64_t> tin(n, -1), low(n, 0);
  std::vector<char> bridge(E, 0);
  struct Frame { uint32_t v; int64_t pe; uint32_t pos; };
  std::vector<Frame> st;
  int64_t timer = 0;
  for (uint32_t s = 0; s < n; ++s) {
    if (tin[s] >= 0 || ofs[s] == ofs[s + 1]) continue;
    tin[s] = low[s] = timer++;
    st.push_back({s, -1, ofs[s]});
    while (!st.empty()) {
      const size_t top = st.size() - 1;
      const uint32_t v = st[top].v;
      if (st[top].pos < ofs[v + 1]) {
        const auto [to, eid] = adj[st[top].pos++];
        if ((int64_t)eid == st[top].pe) continue;
        if (tin[to] >= 0) {
          low[v] = std::min(low[v], tin[to]);
        } else {
          tin[to] = low[to] = timer++;
          st.push_back({to, (int64_t)eid, ofs[to]});
        }
      } else {
        const int64_t pe = st[top].pe;
        st.pop_back();
        if (!st.empty()) {
          const uint32_t p = st.back().v;
          low[p] = std::min(low[p], low[v]);
          if (low[v] > tin[p]) bridge[(size_t)pe] = 1;
        }
      }
    }
  }
  comp.assign(n, -1);
  std::vector<uint32_t> size;
  std::vector<uint32_t> queue;
  for (uint32_t s = 0; s < n; ++s) {
    if (comp[s] >= 0 || ofs[s] == ofs[s + 1]) continue;
    const int c = (int)size.size();
    size.push_back(0);
    comp[s] = c;
    queue.assign(1, s);
    for (size_t h = 0; h < queue.size(); ++h) {
      const uint32_t v = queue[h];
      ++size[c];
      for (uint32_t p = ofs[v]; p < ofs[v + 1]; ++p)
        if (!bridge[adj[p].second] && comp[adj[p].first] < 0) {
          comp[adj[p].first] = c;
          queue.push_back(adj[p].first);
        }
    }
  }
  int best = -1;
  for (size_t c = 0; c < size.size(); ++c)  // components are numbered by their smallest node
    if (size[c] >= 2 && (best < 0 || size[c] > size[(size_t)best])) best = (int)c;
  return best;
}

void incidence_lists(uint32_t m, const std::vector<uint2>& edges, std::vector<uint32_t>& ofs, std::vector<uint32_t>& nbr,
                     std::vector<uint32_t>& edge) {
  const uint32_t ne = (uint32_t)edges.size();
  ofs.assign(m + 1, 0);
  nbr.resize(2 * (size_t)ne);
  edge.resize(2 * (size_t)ne);
  for (const uint2& e : edges) { ofs[e.x + 1]++; ofs[e.y + 1]++; }
  for (uint32_t a = 0; a < m; ++a) ofs[a + 1] += ofs[a];
  std::vector<uint32_t> pos(ofs.begin(), ofs.end() - 1);
  for (uint32_t e = 0; e < ne; ++e) { nbr[pos[edges[e].y]] = edges[e].x; edge[pos[edges[e].y]++] = e; }
  for (uint32_t e = 0; e < ne; ++e) { nbr[pos[edges[e].x]] = edges[e].y; edge[pos[edges[e].x]++] = e; }
}

// the deterministic start of the inverse iteration (the oracle draws the same numbers)
double init_value(uint64_t k) {
  uint64_t z = k * 0x9E3779B97F4A7C15ull + 0x2545F4914F6CDD1Dull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * (1.0 / 9007199254740992.0) - 0.5;
}

int select_component(r3d_ctx* ctx, const char* fn, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                     double max_angular_error_deg, uint8_t* view_kept, uint8_t* edge_kept, uint32_t* edge_support, KeptComponent& K) {
  DeviceWorker& w = ctx->workers[0];
  std::memset(view_kept, 0, n_views);
  if (edge_kept) std::memset(edge_kept, 0, n_rel);
  if (edge_support) std::memset(edge_support, 0, n_rel * sizeof(uint32_t));
  const std::string f(fn);
  // ---- 1. edges: canonical (i < j) with R_ij, checked ----
  struct Edge { uint32_t i, j; uint64_t src; };
  std::vector<Edge> edges;
  for (uint64_t k = 0; k < n_rel; ++k) {
    const r3d_relative_pose& r = rel[k];
    if (r.status != R3D_RELPOSE_OK) continue;
    if (r.I == r.J) return fail(ctx, R3D_ERR_INVALID, f + "an edge joins a view to itself");
    if (r.I >= n_views || r.J >= n_views) return fail(ctx, R3D_ERR_INVALID, f + "view id >= n_views");
    edges.push_back({std::min(r.I, r.J), std::max(r.I, r.J), k});
  }
  K.n_edges = edges.size();
  std::sort(edges.begin(), edges.end(), [](const Edge& a, const Edge& b) { return a.i != b.i ? a.i < b.i : a.j < b.j; });
  for (size_t k = 1; k < edges.size(); ++k)
    if (edges[k].i == edges[k - 1].i && edges[k].j == edges[k - 1].j)
      return fail(ctx, R3D_ERR_INVALID, f + "the same pair of views is given twice");
  if (edges.size() > 0xfffffff0ull) return fail(ctx, R3D_ERR_UNSUPPORTED, f + "too many edges");
  // nodes: the views with an edge, in id order
  std::vector<uint32_t> node_of(n_views, UINT32_MAX), view_of;
  for (const Edge& e : edges) { node_of[e.i] = 0; node_of[e.j] = 0; }
  for (uint32_t v = 0; v < n_views; ++v)
    if (node_of[v] == 0) { node_of[v] = (uint32_t)view_of.size(); view_of.push_back(v); }
  const uint32_t nn = (uint32_t)view_of.size();
  const uint32_t E = (uint32_t)edges.size();
  if (nn > kMaxTripletNodes) return fail(ctx, R3D_ERR_UNSUPPORTED, f + "more than 57344 views with edges");
  // upper CSR over the nodes; edge id = position (edges are sorted by (i, j), so the positions are the sorted order)
  std::vector<uint32_t> up_ofs(nn + 1, 0), up_nbr(E);
  std::vector<double> rot_soa((size_t)9 * E);
  for (uint32_t p = 0; p < E; ++p) {
    const Edge& e = edges[p];
    up_ofs[node_of[e.i] + 1]++;
    up_nbr[p] = node_of[e.j];
    const r3d_relative_pose& r = rel[e.src];
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b)  // R_ij; a reversed entry (I > J) carries R_ji = R_ij^T
        rot_soa[(size_t)(3 * a + b) * E + p] = r.I < r.J ? r.rotation[3 * a + b] : r.rotation[3 * b + a];
  }
  for (uint32_t v = 0; v < nn; ++v) up_ofs[v + 1] += up_ofs[v];
  std::vector<uint32_t> support(E, 0);
  if (E) {
    Events<2> ev;
    R3D_CUDA_TRY(ctx, ev.create());
    DevArr<uint32_t> d_ofs(w), d_nbr(w), d_sup(w), d_work(w);
    DevArr<double> d_rot(w);
    DevArr<unsigned long long> d_cnt(w);
    if (!d_ofs.alloc(nn + 1) || !d_nbr.alloc(E) || !d_sup.alloc(E) || !d_work.alloc(1) || !d_rot.alloc((size_t)9 * E) || !d_cnt.alloc(2))
      return fail(ctx, R3D_ERR_NOMEM, f + "device scratch");
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ofs.p, up_ofs.data(), (nn + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_nbr.p, up_nbr.data(), E * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_rot.p, rot_soa.data(), rot_soa.size() * sizeof(double), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_sup.p, 0, E * sizeof(uint32_t), w.stream));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_work.p, 0, sizeof(uint32_t), w.stream));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_cnt.p, 0, 2 * sizeof(unsigned long long), w.stream));
    const float thr = (float)max_angular_error_deg;
    const double c_thr = std::cos(max_angular_error_deg * (R3D_PI / 180.0));
    const size_t smem = (size_t)nn * sizeof(int32_t);
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_rotavg_triplets, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1)));
    int per_sm = 0;
    R3D_CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rotavg_triplets, kTThreads, smem));
    const uint32_t grid = std::min<uint32_t>(nn, (uint32_t)(w.sm_count * std::max(per_sm, 1)));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[0], w.stream));
    k_rotavg_triplets<<<grid, kTThreads, smem, w.stream>>>(d_ofs.p, d_nbr.p, nn, d_rot.p, E, c_thr - kCycleBand, c_thr + kCycleBand, thr,
                                                          d_work.p, d_sup.p, d_cnt.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[1], w.stream));
    unsigned long long cnt[2];
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(support.data(), d_sup.p, E * sizeof(uint32_t), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(cnt, d_cnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    K.ms_triplets = ev.ms(0, 1);
    K.n_triplets = cnt[0];
    K.n_valid_triplets = cnt[1];
  }
  if (edge_support)
    for (uint32_t p = 0; p < E; ++p) edge_support[edges[p].src] = support[p];
  // ---- 2. largest bi-edge-connected component of the supported edges ----
  std::vector<uint32_t> eu, evv, eid;
  for (uint32_t p = 0; p < E; ++p)
    if (support[p]) { eu.push_back(node_of[edges[p].i]); evv.push_back(up_nbr[p]); eid.push_back(p); }
  std::vector<int> comp;
  const int best = largest_biedge_component(nn, eu, evv, comp);
  if (best < 0) return R3D_OK;
  std::vector<uint32_t> local(nn, UINT32_MAX);  // local index = rank of the view id among the kept views
  for (uint32_t v = 0; v < nn; ++v)
    if (comp[v] == best) { local[v] = (uint32_t)K.kview.size(); K.kview.push_back(view_of[v]); }
  const uint32_t m = (uint32_t)K.kview.size();
  if (m > R3D_ROTAVG_MAX_VIEWS) {
    K.kview.clear();
    return fail(ctx, R3D_ERR_UNSUPPORTED, f + "more than R3D_ROTAVG_MAX_VIEWS views in the component");
  }
  for (size_t q = 0; q < eid.size(); ++q) {
    const uint32_t p = eid[q];
    const uint32_t a = local[eu[q]], b = local[evv[q]];
    if (a == UINT32_MAX || b == UINT32_MAX) continue;
    K.kab.push_back(make_uint2(a, b));
    for (int c = 0; c < 9; ++c) K.kR.push_back(rot_soa[(size_t)c * E + p]);
    if (edge_kept) edge_kept[edges[p].src] = 1;
  }
  for (uint32_t v : K.kview) view_kept[v] = 1;
  incidence_lists(m, K.kab, K.inc_ofs, K.inc_nbr, K.inc_edge);
  return R3D_OK;
}

int rotation_averaging(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views, const r3d_rotavg_options& opt,
                       double* rotations, uint8_t* view_kept, uint8_t* edge_kept, uint32_t* edge_support, r3d_rotavg_summary& S) {
  const double t0 = now_ms();
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::memset(rotations, 0, (size_t)n_views * 9 * sizeof(double));
  S.lm_termination = -1;
  // ---- 1, 2. the kept component ----
  KeptComponent K;
  int rc = select_component(ctx, "r3d_rotation_averaging: ", rel, n_rel, n_views, opt.max_angular_error_deg, view_kept, edge_kept,
                            edge_support, K);
  S.n_edges = K.n_edges;
  S.n_triplets = K.n_triplets;
  S.n_valid_triplets = K.n_valid_triplets;
  S.ms_triplets = K.ms_triplets;
  if (rc) return rc;
  if (K.kview.empty()) {
    S.success = 0;
    S.ms_device_total = S.ms_triplets;
    S.ms_host = now_ms() - t0 - S.ms_device_total;
    return R3D_OK;
  }
  const std::vector<uint32_t>& kview = K.kview;
  const std::vector<uint2>& kab = K.kab;
  const std::vector<double>& kR = K.kR;
  const std::vector<uint32_t>&inc_ofs = K.inc_ofs, &inc_nbr = K.inc_nbr, &inc_edge = K.inc_edge;
  const uint32_t m = (uint32_t)kview.size();
  const uint32_t ne = (uint32_t)kab.size();
  S.success = 1;
  S.n_kept_views = m;
  S.n_kept_edges = ne;
  Events<6> ev;
  R3D_CUDA_TRY(ctx, ev.create());
  uint32_t max_deg = 0;
  for (uint32_t a = 0; a < m; ++a) max_deg = std::max(max_deg, inc_ofs[a + 1] - inc_ofs[a]);
  // ---- 3. L2 initialisation ----
  const int N = 3 * (int)m;
  const int nblk = (N + kCholNB - 1) / kCholNB;
  DevArr<uint32_t> d_iofs(w), d_inbr(w), d_iedge(w);
  DevArr<uint2> d_ab(w);
  DevArr<double> d_R(w), d_A(w), d_L(w), d_Linv(w), d_x(w), d_Y(w), d_Z(w), d_Q(w), d_Rout(w), d_scal(w);
  if (!d_iofs.alloc(m + 1) || !d_inbr.alloc(2 * (size_t)ne) || !d_iedge.alloc(2 * (size_t)ne) || !d_ab.alloc(ne) || !d_R.alloc(9 * (size_t)ne) ||
      !d_A.alloc((size_t)(N + 1) * N) || !d_L.alloc((size_t)(N + 1) * N + 64) || !d_Linv.alloc((size_t)nblk * kCholNB * kCholNB) ||
      !d_x.alloc(N) || !d_Y.alloc(3 * (size_t)N) || !d_Z.alloc(3 * (size_t)N) || !d_Q.alloc(3 * (size_t)N) || !d_Rout.alloc(9 * (size_t)m) ||
      !d_scal.alloc(8))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_rotation_averaging: device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_iofs.p, inc_ofs.data(), (m + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_inbr.p, inc_nbr.data(), inc_nbr.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_iedge.p, inc_edge.data(), inc_edge.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ab.p, kab.data(), kab.size() * sizeof(uint2), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_R.p, kR.data(), kR.size() * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  std::vector<double> y0(3 * (size_t)N);
  for (size_t k = 0; k < y0.size(); ++k) y0[k] = init_value(k);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_Y.p, y0.data(), y0.size() * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  double scal[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  auto read_scal = [&]() -> int {
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(scal, d_scal.p, sizeof(scal), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    return R3D_OK;
  };
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[2], w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_A.p, 0, (size_t)(N + 1) * N * sizeof(double), w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_scal.p, 0, 8 * sizeof(double), w.stream));
  {
    const uint32_t nt = std::max<uint32_t>(m, 2 * ne);
    k_rotavg_assemble_M<<<(nt + 255) / 256, 256, 0, w.stream>>>(d_iofs.p, d_inbr.p, d_iedge.p, d_R.p, m, kSigmaRel * (double)max_deg, d_A.p);
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  if ((rc = dense_cholesky(ctx, w, d_A.p, d_L.p, d_Linv.p, N, d_scal.p + 7, d_x.p))) return rc;
  k_rotavg_orth<<<1, kOThreads, 0, w.stream>>>(d_Y.p, d_Q.p, N, 1, d_scal.p);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  if ((rc = read_scal())) return rc;
  if (scal[7] != 0.0) return fail(ctx, R3D_ERR_CUDA, "r3d_rotation_averaging: M + sigma I is not positive definite");
  int trsm_grid = 0;
  if ((rc = trsm3_grid(ctx, w, &trsm_grid))) return rc;
  uint32_t it = 0;
  for (; it < kInitMaxIter;) {
    ++it;
    if ((rc = trsm3(ctx, w, d_L.p, d_Linv.p, N, d_Y.p, d_Z.p, trsm_grid))) return rc;
    k_rotavg_orth<<<1, kOThreads, 0, w.stream>>>(d_Y.p, d_Q.p, N, 0, d_scal.p);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if ((rc = read_scal())) return rc;
    if (!(scal[0] >= kInitTol)) break;  // converged (or NaN: stop, the projection shows it)
  }
  S.init_iterations = it;
  k_rotavg_project<<<1, kOThreads, 0, w.stream>>>(d_Q.p, m, d_Rout.p);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[3], w.stream));
  std::vector<double> Rl(9 * (size_t)m);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(Rl.data(), d_Rout.p, Rl.size() * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  S.ms_init = ev.ms(2, 3);
  // ---- 4. refinement ----
  if (opt.refine) {
    std::vector<double> aa(3 * (size_t)m);
    for (uint32_t a = 0; a < m; ++a) rp::rotation_to_angle_axis(&Rl[9 * (size_t)a], &aa[3 * (size_t)a]);
    DevArr<double> d_aa(w), d_aan(w), d_res(w), d_jac(w), d_cost(w), d_scale(w), d_g(w), d_diag(w);
    if (!d_aa.alloc(N) || !d_aan.alloc(N) || !d_res.alloc(3 * (size_t)ne) || !d_jac.alloc(18 * (size_t)ne) || !d_cost.alloc(ne) ||
        !d_scale.alloc(N) || !d_g.alloc(N) || !d_diag.alloc(N))
      return fail(ctx, R3D_ERR_NOMEM, "r3d_rotation_averaging: device scratch");
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_aa.p, aa.data(), N * sizeof(double), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[4], w.stream));
    const double ha = opt.lm.huber_a;
    const uint32_t eg = (ne + 127) / 128;
    double* cur = d_aa.p;
    double* trial = d_aan.p;
    const AvgBuffers B{d_iofs.p, d_iedge.p, d_ab.p, d_res.p, d_jac.p, d_cost.p, d_scale.p, d_g.p, d_diag.p,
                       d_A.p, d_L.p, d_Linv.p, d_x.p, d_scal.p};
    rc = averaging_lm<18>(
        ctx, w, lm_params(opt.lm), B, ne, 0, (uint32_t)N, (uint32_t)N, cur, trial, S,
        [&](const double* x) { k_rotavg_cost<<<eg, 128, 0, w.stream>>>(x, d_ab.p, d_R.p, ne, ha, d_cost.p); },
        [&](const double* x) { k_rotavg_eval<<<eg, 128, 0, w.stream>>>(x, d_ab.p, d_R.p, ne, ha, d_res.p, d_jac.p); },
        [](int) {},
        [&](const double*, double inv_radius) {
          k_rotavg_system<<<m, 128, 0, w.stream>>>(d_iofs.p, d_inbr.p, d_iedge.p, d_ab.p, d_jac.p, m, d_scale.p, d_g.p, d_diag.p,
                                                   inv_radius, d_A.p);
        },
        [](const double*, double) {});
    if (rc) return rc;
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[5], w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(aa.data(), cur, N * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    S.ms_refine = ev.ms(4, 5);
    // back to matrices, the gauge again
    std::vector<double> R0(9);
    rp::angle_axis_to_rotation(&aa[0], R0.data());
    for (uint32_t a = 0; a < m; ++a) {
      double R[9];
      rp::angle_axis_to_rotation(&aa[3 * (size_t)a], R);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
          Rl[9 * (size_t)a + 3 * r + c] = a == 0 ? (r == c ? 1.0 : 0.0) : R[3 * r] * R0[3 * c] + R[3 * r + 1] * R0[3 * c + 1] + R[3 * r + 2] * R0[3 * c + 2];
    }
  }
  for (uint32_t a = 0; a < m; ++a) std::memcpy(rotations + 9 * (size_t)kview[a], &Rl[9 * (size_t)a], 9 * sizeof(double));
  S.ms_device_total = S.ms_triplets + S.ms_init + S.ms_refine;
  S.ms_host = now_ms() - t0 - S.ms_device_total;
  return R3D_OK;
}

}  // namespace ra
}  // namespace r3d

using namespace r3d;

extern "C" void r3d_rotavg_default_options(r3d_rotavg_options* o) {
  if (!o) return;
  o->method = R3D_ROTAVG_L2;
  o->max_angular_error_deg = 5.0;  // TripletRotationRejection(5.0, ...)
  o->refine = 1;
  r3d_ba_default_options(&o->lm);
  o->lm.huber_a = 0.0;             // L2RotationAveraging_Refine: no loss function
  o->lm.refine_intrinsics = 0;
}

extern "C" int r3d_rotation_averaging(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                                      const r3d_rotavg_options* opt, double* rotations, uint8_t* view_kept, uint8_t* edge_kept,
                                      uint32_t* edge_support, r3d_rotavg_summary* summary) {
  if (!ctx || (!rel && n_rel) || !opt || (!rotations && n_views) || (!view_kept && n_views) || !summary)
    return fail(ctx, R3D_ERR_INVALID, "r3d_rotation_averaging: bad arguments");
  std::memset(summary, 0, sizeof(*summary));
  summary->lm_termination = -1;
  if (opt->method == R3D_ROTAVG_L1) return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_rotation_averaging: L1 rotation averaging is not implemented");
  if (opt->method != R3D_ROTAVG_L2) return fail(ctx, R3D_ERR_INVALID, "r3d_rotation_averaging: unknown method");
  if (!(opt->max_angular_error_deg > 0.0)) return fail(ctx, R3D_ERR_INVALID, "r3d_rotation_averaging: max_angular_error_deg <= 0");
  return ra::rotation_averaging(ctx, rel, n_rel, n_views, *opt, rotations, view_kept, edge_kept, edge_support, *summary);
}

extern "C" int r3d_debug_chol_solve3(r3d_ctx* ctx, int n, const double* A, const double* Y, int grid, double* X_out) {
  if (!ctx || n < 1 || !A || !Y || !X_out || grid < 0) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_chol_solve3: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  int rc;
  if ((rc = ra::trsm3_grid(ctx, w, &grid))) return rc;
  const int nblk = (n + kCholNB - 1) / kCholNB;
  // as rotation_averaging allocates them: M | unused rhs row, L with the slack of dense_cholesky's contract
  DevArr<double> d_A(w), d_L(w), d_Linv(w), d_x(w), d_Y(w), d_Z(w), d_flag(w);
  if (!d_A.alloc((size_t)(n + 1) * n) || !d_L.alloc((size_t)(n + 1) * n + 64) || !d_Linv.alloc((size_t)nblk * kCholNB * kCholNB) ||
      !d_x.alloc(n) || !d_Y.alloc(3 * (size_t)n) || !d_Z.alloc(3 * (size_t)n) || !d_flag.alloc(1))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_debug_chol_solve3: device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_A.p, A, (size_t)n * n * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_A.p + (size_t)n * n, 0, (size_t)n * sizeof(double), w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_Y.p, Y, 3 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_flag.p, 0, sizeof(double), w.stream));
  if ((rc = dense_cholesky(ctx, w, d_A.p, d_L.p, d_Linv.p, n, d_flag.p, d_x.p))) return rc;
  if ((rc = ra::trsm3(ctx, w, d_L.p, d_Linv.p, n, d_Y.p, d_Z.p, grid))) return rc;
  double flag = 0.0;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(&flag, d_flag.p, sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(X_out, d_Y.p, 3 * (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  if (flag != 0.0) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_chol_solve3: A is not positive definite");
  return R3D_OK;
}

extern "C" int r3d_matches_keep_largest_biedge_component(const r3d_matches* m, r3d_matches** out) {
  if (!m || !out) return R3D_ERR_INVALID;
  *out = nullptr;
  const size_t P = m->pairs.size() / 2;
  std::vector<uint32_t> ids(m->pairs.begin(), m->pairs.end());
  std::sort(ids.begin(), ids.end());
  ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
  auto node = [&](uint32_t v) { return (uint32_t)(std::lower_bound(ids.begin(), ids.end(), v) - ids.begin()); };
  std::vector<uint32_t> eu(P), ev(P);
  for (size_t p = 0; p < P; ++p) { eu[p] = node(m->pairs[2 * p]); ev[p] = node(m->pairs[2 * p + 1]); }
  std::vector<int> comp;
  const int best = ra::largest_biedge_component((uint32_t)ids.size(), eu, ev, comp);
  r3d_matches* r = new r3d_matches();
  r->slabs = m->slabs;
  if (best >= 0)
    for (size_t p = 0; p < P; ++p)
      if (comp[eu[p]] == best && comp[ev[p]] == best) r->push_span(m->pairs[2 * p], m->pairs[2 * p + 1], m->per[p]);
  *out = r;
  return R3D_OK;
}
