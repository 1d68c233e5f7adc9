// oracle_rotavg.cpp -- CPU ORACLE (test infrastructure; see oracle_rotavg.h), liboracle_rotavg.so (oracle/rotavg.mk).
//
// Restates GlobalSfM_Rotation_AveragingSolver::Run with ROTATION_AVERAGING_L2, the second step of the global pipeline
// (GlobalSfMReconstructionEngine_RelativeMotions::Compute_Global_Rotations, reached from
// src/threads/R3DTriangulationThread.cpp:201-250; un-vendored OpenMVG 1.4, SURVEY.md A.10):
//   * one edge (I, J) with R_IJ per OK relative pose, R_J ~ R_IJ R_I, weight 1;
//   * TripletListing + TripletRotationRejection(5.0): every triangle i < j < k, cycle R_ki R_jk R_ij, error
//     float(R2D(acos(clamp((trace - 1) / 2, -1, 1)))) < threshold, the acos of oracle_detmath.hpp; an edge survives
//     when a valid triangle holds it;
//   * CleanGraph_KeepLargestBiEdge_Nodes + KeepOnlyReferencedElement: bridges by Tarjan's low-link, the connected
//     components of the rest, the one with the most nodes (tie: the one with the smallest view id);
//   * L2RotationAveraging (Martinec-Pajdla): the 3 smallest eigenvectors of M = A^T A by block inverse iteration on
//     M + sigma I (dense Cholesky, 3 right-hand sides, 3 x 3 Cholesky-QR), sign by sum det, SO(3) projection of every
//     block with the oracle's Jacobi SVD, gauge R = I on the lowest kept view id;
//   * L2RotationAveraging_Refine: angle-axis per view, residual log(R_ij^T R_j R_i^T) by forward-mode autodiff (Ceres'
//     AngleAxisToRotationMatrix / RotationMatrixToAngleAxis on jets), the trust-region LM of oracle_ba.cpp (SURVEY.md
//     A.7) on the dense normal equations; the gauge again.
// Deliberate, documented deviations (DESIGN.md sec. 2): inverse iteration instead of Eigen::SelfAdjointEigenSolver, the
// Jacobi SVD instead of Eigen::JacobiSVD, the explicit gauge.
// PARITY UNPINNED.
#include "oracle_rotavg.h"
#include "oracle_detmath.hpp"

#include <algorithm>
#include <array>
#include <cmath>
#include <limits>
#include <cstring>
#include <vector>
#include <omp.h>

namespace orc {
namespace rp {  // oracle_relpose.cpp (liboracle_relpose.so)
void svd3(const double* A, double* U, double* S, double* V);
double det3(const double* M);
void rotation_to_angle_axis(const double* R, double* aa);
void angle_axis_to_rotation(const double* aa, double* R);
}  // namespace rp

namespace ra {

const double kSigmaRel = 1e-7;
const double kInitTol = 1e-12;
const uint32_t kInitMaxIter = 100;

// ---- triplets ----
double cycle_trace(const double* Rij, const double* Rjk, const double* Rik) {
  double tr = 0.0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      const double t = Rjk[3 * a] * Rij[b] + Rjk[3 * a + 1] * Rij[3 + b] + Rjk[3 * a + 2] * Rij[6 + b];
      tr = tr + Rik[3 * a + b] * t;
    }
  return tr;
}
float cycle_error_deg(const double* Rij, const double* Rjk, const double* Rik) {
  double c = (cycle_trace(Rij, Rjk, Rik) - 1.0) / 2.0;
  c = std::min(1.0, std::max(-1.0, c));
  return (float)(det::acos(c) / det::kPi * 180.0);
}

// ---- graph ----
int largest_biedge_component(uint32_t n, const std::vector<uint32_t>& eu, const std::vector<uint32_t>& ev, std::vector<int>& comp) {
  std::vector<std::vector<std::pair<uint32_t, uint32_t>>> adj(n);
  for (size_t k = 0; k < eu.size(); ++k)
    if (eu[k] != ev[k]) {
      adj[eu[k]].push_back({ev[k], (uint32_t)k});
      adj[ev[k]].push_back({eu[k], (uint32_t)k});
    }
  std::vector<long> tin(n, -1), low(n, 0);
  std::vector<char> bridge(eu.size(), 0);
  long timer = 0;
  // iterative DFS: a stack of (node, parent edge, next neighbour)
  std::vector<std::array<long, 3>> st;
  for (uint32_t s = 0; s < n; ++s) {
    if (tin[s] >= 0 || adj[s].empty()) continue;
    tin[s] = low[s] = timer++;
    st.push_back({(long)s, -1, 0});
    while (!st.empty()) {
      std::array<long, 3>& f = st.back();
      const uint32_t v = (uint32_t)f[0];
      if (f[2] < (long)adj[v].size()) {
        const auto nb = adj[v][(size_t)f[2]++];
        if ((long)nb.second == f[1]) continue;
        if (tin[nb.first] >= 0) {
          low[v] = std::min(low[v], tin[nb.first]);
        } else {
          tin[nb.first] = low[nb.first] = timer++;
          st.push_back({(long)nb.first, (long)nb.second, 0});
        }
      } else {
        const long pe = f[1];
        st.pop_back();
        if (!st.empty()) {
          const uint32_t p = (uint32_t)st.back()[0];
          low[p] = std::min(low[p], low[v]);
          if (low[v] > tin[p]) bridge[(size_t)pe] = 1;
        }
      }
    }
  }
  comp.assign(n, -1);
  std::vector<uint32_t> size;
  for (uint32_t s = 0; s < n; ++s) {
    if (comp[s] >= 0 || adj[s].empty()) continue;
    const int c = (int)size.size();
    size.push_back(0);
    std::vector<uint32_t> stack(1, s);
    comp[s] = c;
    while (!stack.empty()) {
      const uint32_t v = stack.back();
      stack.pop_back();
      ++size[c];
      for (const auto& nb : adj[v])
        if (!bridge[nb.second] && comp[nb.first] < 0) {
          comp[nb.first] = c;
          stack.push_back(nb.first);
        }
    }
  }
  int best = -1;
  for (size_t c = 0; c < size.size(); ++c)
    if (size[c] >= 2 && (best < 0 || size[c] > size[(size_t)best])) best = (int)c;
  return best;
}

// ---- dense SPD ----
// in place lower Cholesky of an n x n row-major matrix; false if not positive definite
bool cholesky(std::vector<double>& A, int n, int n_threads) {
  for (int j = 0; j < n; ++j) {
    double d = A[(size_t)j * n + j];
    for (int t = 0; t < j; ++t) d -= A[(size_t)j * n + t] * A[(size_t)j * n + t];
    if (!(d > 0.0)) return false;
    d = std::sqrt(d);
    A[(size_t)j * n + j] = d;
#pragma omp parallel for schedule(static) num_threads(n_threads) if (n - j > 256)
    for (int i = j + 1; i < n; ++i) {
      double s = A[(size_t)i * n + j];
      const double* ai = &A[(size_t)i * n];
      const double* aj = &A[(size_t)j * n];
      for (int t = 0; t < j; ++t) s -= ai[t] * aj[t];
      A[(size_t)i * n + j] = s / d;
    }
  }
  return true;
}
// L L^T x = b for k right-hand sides (b: n x k row-major), in place
void chol_solve(const std::vector<double>& L, int n, double* b, int k) {
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < k; ++c) {
      double s = b[(size_t)i * k + c];
      for (int t = 0; t < i; ++t) s -= L[(size_t)i * n + t] * b[(size_t)t * k + c];
      b[(size_t)i * k + c] = s / L[(size_t)i * n + i];
    }
  for (int i = n - 1; i >= 0; --i)
    for (int c = 0; c < k; ++c) {
      double s = b[(size_t)i * k + c];
      for (int t = i + 1; t < n; ++t) s -= L[(size_t)t * n + i] * b[(size_t)t * k + c];
      b[(size_t)i * k + c] = s / L[(size_t)i * n + i];
    }
}

double init_value(uint64_t k) {  // the device's start (rotavg.cu)
  uint64_t z = k * 0x9E3779B97F4A7C15ull + 0x2545F4914F6CDD1Dull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * (1.0 / 9007199254740992.0) - 0.5;
}

// orthonormalise the columns of Y (n x 3) by Cholesky-QR
void cholqr3(std::vector<double>& Y, int n) {
  double g[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < n; ++i) {
    const double* y = &Y[3 * (size_t)i];
    g[0] += y[0] * y[0]; g[1] += y[1] * y[0]; g[2] += y[1] * y[1]; g[3] += y[2] * y[0]; g[4] += y[2] * y[1]; g[5] += y[2] * y[2];
  }
  const double l00 = std::sqrt(g[0]), l10 = g[1] / l00, l20 = g[3] / l00;
  const double l11 = std::sqrt(g[2] - l10 * l10), l21 = (g[4] - l20 * l10) / l11;
  const double l22 = std::sqrt(g[5] - l20 * l20 - l21 * l21);
  for (int i = 0; i < n; ++i) {  // y L^-T by substitution
    double* y = &Y[3 * (size_t)i];
    const double q0 = y[0] / l00;
    const double q1 = (y[1] - l10 * q0) / l11;
    const double q2 = (y[2] - l20 * q0 - l21 * q1) / l22;
    y[0] = q0; y[1] = q1; y[2] = q2;
  }
}

// M = A^T A + sigma I of the kept edges (local ids a < b, R_ab), dense N x N
void assemble_M(const std::vector<uint32_t>& ab, const std::vector<double>& R, uint32_t m, std::vector<double>& M, double* sigma_out) {
  const int N = 3 * (int)m;
  M.assign((size_t)N * N, 0.0);
  std::vector<uint32_t> deg(m, 0);
  for (size_t e = 0; e < ab.size() / 2; ++e) { deg[ab[2 * e]]++; deg[ab[2 * e + 1]]++; }
  const double sigma = kSigmaRel * (double)*std::max_element(deg.begin(), deg.end());
  for (size_t e = 0; e < ab.size() / 2; ++e) {
    const uint32_t a = ab[2 * e], b = ab[2 * e + 1];
    const double* Re = &R[9 * e];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        M[(size_t)(3 * a + r) * N + 3 * b + c] = -Re[3 * c + r];
        M[(size_t)(3 * b + r) * N + 3 * a + c] = -Re[3 * r + c];
      }
  }
  for (uint32_t a = 0; a < m; ++a)
    for (int r = 0; r < 3; ++r) M[(size_t)(3 * a + r) * N + 3 * a + r] = (double)deg[a] + sigma;
  if (sigma_out) *sigma_out = sigma;
}

// the 3 smallest eigenvectors of M (orthonormal columns of Q, N x 3); returns the iteration count, 0 if not PD
uint32_t l2_subspace(const std::vector<uint32_t>& ab, const std::vector<double>& R, uint32_t m, std::vector<double>& Q, int n_threads) {
  const int N = 3 * (int)m;
  std::vector<double> L;
  assemble_M(ab, R, m, L, nullptr);
  if (!cholesky(L, N, n_threads)) return 0;
  Q.resize(3 * (size_t)N);
  for (size_t k = 0; k < Q.size(); ++k) Q[k] = init_value(k);
  cholqr3(Q, N);
  std::vector<double> Y;
  uint32_t it = 0;
  while (it < kInitMaxIter) {
    ++it;
    Y = Q;
    chol_solve(L, N, Y.data(), 3);
    cholqr3(Y, N);
    double C[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < N; ++i)
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) C[3 * a + b] += Q[3 * (size_t)i + a] * Y[3 * (size_t)i + b];
    double ch = 0.0;
    for (int i = 0; i < N; ++i)
      for (int b = 0; b < 3; ++b) {
        const double d = Y[3 * (size_t)i + b] - (Q[3 * (size_t)i] * C[b] + Q[3 * (size_t)i + 1] * C[3 + b] + Q[3 * (size_t)i + 2] * C[6 + b]);
        ch += d * d;
      }
    Q.swap(Y);
    if (!(std::sqrt(ch) >= kInitTol)) break;
  }
  return it;
}

void project_so3(const double* X, double* R) {
  double U[9], S[3], V[9];
  rp::svd3(X, U, S, V);
  V[2] = V[3] * V[7] - V[6] * V[4];
  V[5] = V[6] * V[1] - V[0] * V[7];
  V[8] = V[0] * V[4] - V[3] * V[1];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[3 * r + c] = U[3 * r] * V[3 * c] + U[3 * r + 1] * V[3 * c + 1] + U[3 * r + 2] * V[3 * c + 2];
}

// R_i <- R_i R_0^T, R_0 = I
void apply_gauge(std::vector<double>& Rl, uint32_t m) {
  const std::vector<double> R0(Rl.begin(), Rl.begin() + 9);
  for (uint32_t a = 0; a < m; ++a) {
    double R[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        R[3 * r + c] = a == 0 ? (r == c ? 1.0 : 0.0)
                              : Rl[9 * a + 3 * r] * R0[3 * c] + Rl[9 * a + 3 * r + 1] * R0[3 * c + 1] + Rl[9 * a + 3 * r + 2] * R0[3 * c + 2];
    std::memcpy(&Rl[9 * (size_t)a], R, sizeof(R));
  }
}

// ---- refinement: jets ----
struct Jet {
  double a;
  double v[6];
};
Jet jc(double x) { Jet r; r.a = x; for (int i = 0; i < 6; ++i) r.v[i] = 0.0; return r; }
Jet operator+(const Jet& x, const Jet& y) { Jet r; r.a = x.a + y.a; for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
Jet operator-(const Jet& x, const Jet& y) { Jet r; r.a = x.a - y.a; for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
Jet operator-(const Jet& x) { Jet r; r.a = -x.a; for (int i = 0; i < 6; ++i) r.v[i] = -x.v[i]; return r; }
Jet operator*(const Jet& x, const Jet& y) { Jet r; r.a = x.a * y.a; for (int i = 0; i < 6; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
Jet operator/(const Jet& x, const Jet& y) { Jet r; const double inv = 1.0 / y.a; r.a = x.a * inv; for (int i = 0; i < 6; ++i) r.v[i] = (x.v[i] - r.a * y.v[i]) * inv; return r; }
Jet operator+(const Jet& x, double s) { Jet r = x; r.a += s; return r; }
Jet operator-(double s, const Jet& x) { Jet r = -x; r.a += s; return r; }
Jet operator*(double s, const Jet& x) { Jet r; r.a = x.a * s; for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] * s; return r; }
Jet sqrt(const Jet& x) { Jet r; r.a = std::sqrt(x.a); const double d = 0.5 / r.a; for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] * d; return r; }
Jet sin(const Jet& x) { Jet r; r.a = std::sin(x.a); const double c = std::cos(x.a); for (int i = 0; i < 6; ++i) r.v[i] = c * x.v[i]; return r; }
Jet cos(const Jet& x) { Jet r; r.a = std::cos(x.a); const double s = -std::sin(x.a); for (int i = 0; i < 6; ++i) r.v[i] = s * x.v[i]; return r; }
Jet atan2(const Jet& y, const Jet& x) {
  Jet r; r.a = std::atan2(y.a, x.a); const double d = 1.0 / (x.a * x.a + y.a * y.a);
  for (int i = 0; i < 6; ++i) r.v[i] = (x.a * y.v[i] - y.a * x.v[i]) * d;
  return r;
}
double sqrt(double x) { return std::sqrt(x); }
double sin(double x) { return std::sin(x); }
double cos(double x) { return std::cos(x); }
double atan2(double y, double x) { return std::atan2(y, x); }
double val(const Jet& x) { return x.a; }
double val(double x) { return x; }
template <class T> T mk(double x);
template <> double mk<double>(double x) { return x; }
template <> Jet mk<Jet>(double x) { return jc(x); }

template <class T>
void aa_to_R(const T* aa, T* R) {  // ceres::AngleAxisToRotationMatrix
  const T th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (val(th2) > 2.220446049250313e-16) {
    const T th = sqrt(th2);
    const T wx = aa[0] / th, wy = aa[1] / th, wz = aa[2] / th;
    const T c = cos(th), s = sin(th), oc = 1.0 - c;
    R[0] = c + wx * wx * oc;      R[1] = wx * wy * oc - wz * s; R[2] = wy * s + wx * wz * oc;
    R[3] = wz * s + wx * wy * oc; R[4] = c + wy * wy * oc;      R[5] = wy * wz * oc - wx * s;
    R[6] = wx * wz * oc - wy * s; R[7] = wx * s + wy * wz * oc; R[8] = c + wz * wz * oc;
  } else {
    R[0] = mk<T>(1.0); R[1] = -aa[2];     R[2] = aa[1];
    R[3] = aa[2];      R[4] = mk<T>(1.0); R[5] = -aa[0];
    R[6] = -aa[1];     R[7] = aa[0];      R[8] = mk<T>(1.0);
  }
}
template <class T>
void R_to_aa(const T* R, T* aa) {  // ceres::RotationMatrixToAngleAxis (quaternion route)
  T q[4];
  const T tr = R[0] + R[4] + R[8];
  if (val(tr) >= 0.0) {
    T t = sqrt(tr + 1.0);
    q[0] = 0.5 * t;
    t = mk<T>(0.5) / t;
    q[1] = (R[7] - R[5]) * t;
    q[2] = (R[2] - R[6]) * t;
    q[3] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (val(R[4]) > val(R[0])) i = 1;
    if (val(R[8]) > val(R[4 * i])) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    T t = sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i + 1] = 0.5 * t;
    t = mk<T>(0.5) / t;
    q[0] = (R[3 * k + j] - R[3 * j + k]) * t;
    q[j + 1] = (R[3 * j + i] + R[3 * i + j]) * t;
    q[k + 1] = (R[3 * k + i] + R[3 * i + k]) * t;
  }
  const T s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (val(s2) > 0.0) {
    const T st = sqrt(s2);
    const T two_theta = 2.0 * (val(q[0]) < 0.0 ? atan2(-st, -q[0]) : atan2(st, q[0]));
    const T kk = two_theta / st;
    for (int c = 0; c < 3; ++c) aa[c] = q[c + 1] * kk;
  } else {
    for (int c = 0; c < 3; ++c) aa[c] = 2.0 * q[c + 1];
  }
}
// r = log(R_ab^T R_b R_a^T)
template <class T>
void edge_residual(const T* aa_a, const T* aa_b, const double* Rab, T* r) {
  T Ra[9], Rb[9], P[9], E[9];
  aa_to_R(aa_a, Ra);
  aa_to_R(aa_b, Rb);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) P[3 * i + j] = Rb[3 * i] * Ra[3 * j] + Rb[3 * i + 1] * Ra[3 * j + 1] + Rb[3 * i + 2] * Ra[3 * j + 2];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[3 * i + j] = Rab[i] * P[j] + Rab[3 + i] * P[3 + j] + Rab[6 + i] * P[6 + j];
  R_to_aa(E, r);
}

double huber_rho(double s, double a, double* rho1) {  // oracle_ba.cpp
  if (a <= 0) { *rho1 = 1.0; return s; }
  const double b = a * a;
  if (s > b) {
    const double rr = std::sqrt(s);
    *rho1 = std::max(std::numeric_limits<double>::min(), a / rr);
    return 2.0 * a * rr - b;
  }
  *rho1 = 1.0;
  return s;
}

struct Refine {
  const std::vector<uint32_t>& ab;
  const std::vector<double>& R;
  uint32_t m;
  double huber_a;
  int n_threads;
  size_t ne() const { return ab.size() / 2; }
  double cost(const std::vector<double>& aa) const {
    std::vector<double> c(ne());
#pragma omp parallel for schedule(static) num_threads(n_threads)
    for (int64_t e = 0; e < (int64_t)ne(); ++e) {
      double r[3], rho1;
      edge_residual(&aa[3 * (size_t)ab[2 * e]], &aa[3 * (size_t)ab[2 * e + 1]], &R[9 * (size_t)e], r);
      c[(size_t)e] = 0.5 * huber_rho(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], huber_a, &rho1);
    }
    double s = 0.0;
    for (double v : c) s += v;
    return s;
  }
};

int run_l2(const std::vector<uint32_t>& ab, const std::vector<double>& R, uint32_t m, const orc_rotavg_options& o, std::vector<double>& Rl,
           orc_rotavg_summary& S, int n_threads) {
  const int N = 3 * (int)m;
  std::vector<double> Q;
  S.init_iterations = l2_subspace(ab, R, m, Q, n_threads);
  if (S.init_iterations == 0) return -2;
  double ds = 0.0;
  for (uint32_t a = 0; a < m; ++a) ds += rp::det3(&Q[9 * (size_t)a]);
  const double sg = ds < 0.0 ? -1.0 : 1.0;
  Rl.assign(9 * (size_t)m, 0.0);
  for (uint32_t a = 0; a < m; ++a) {
    double X[9];
    for (int k = 0; k < 9; ++k) X[k] = sg * Q[9 * (size_t)a + k];
    project_so3(X, &Rl[9 * (size_t)a]);
  }
  apply_gauge(Rl, m);
  if (!o.refine) return 0;
  // ---- Levenberg-Marquardt (oracle_ba.cpp's state machine) ----
  const orc_ba_options& lm = o.lm;
  Refine P{ab, R, m, lm.huber_a, n_threads};
  const size_t ne = P.ne();
  std::vector<double> aa(N), aa_new(N);
  for (uint32_t a = 0; a < m; ++a) rp::rotation_to_angle_axis(&Rl[9 * (size_t)a], &aa[3 * (size_t)a]);
  std::vector<double> res(3 * ne), jac(18 * ne), scale(N, 1.0), g(N), diag(N), delta(N);
  bool have_scale = false;
  auto evaluate = [&]() {
#pragma omp parallel for schedule(static) num_threads(n_threads)
    for (int64_t e = 0; e < (int64_t)ne; ++e) {
      Jet xa[3], xb[3], r[3];
      for (int k = 0; k < 3; ++k) {
        xa[k] = jc(aa[3 * (size_t)ab[2 * e] + k]);
        xa[k].v[k] = 1.0;
        xb[k] = jc(aa[3 * (size_t)ab[2 * e + 1] + k]);
        xb[k].v[3 + k] = 1.0;
      }
      edge_residual(xa, xb, &R[9 * (size_t)e], r);
      double rho1;
      huber_rho(r[0].a * r[0].a + r[1].a * r[1].a + r[2].a * r[2].a, lm.huber_a, &rho1);
      const double sq = std::sqrt(rho1);
      for (int i = 0; i < 3; ++i) {
        res[3 * (size_t)e + i] = r[i].a * sq;
        for (int k = 0; k < 6; ++k) jac[18 * (size_t)e + 6 * i + k] = r[i].v[k] * sq;
      }
    }
    if (!have_scale) {
      std::vector<double> n2(N, 0.0);
      for (size_t e = 0; e < ne; ++e)
        for (int i = 0; i < 3; ++i)
          for (int k = 0; k < 6; ++k) {
            const size_t col = 3 * (size_t)ab[2 * e + (k / 3)] + k % 3;
            n2[col] += jac[18 * e + 6 * i + k] * jac[18 * e + 6 * i + k];
          }
      for (int j = 0; j < N; ++j) scale[j] = 1.0 / (1.0 + std::sqrt(n2[j]));
      have_scale = true;
    }
    for (size_t e = 0; e < ne; ++e)
      for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 6; ++k) jac[18 * e + 6 * i + k] *= scale[3 * (size_t)ab[2 * e + (k / 3)] + k % 3];
    std::fill(g.begin(), g.end(), 0.0);
    std::fill(diag.begin(), diag.end(), 0.0);
    for (size_t e = 0; e < ne; ++e)
      for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 6; ++k) {
          const size_t col = 3 * (size_t)ab[2 * e + (k / 3)] + k % 3;
          g[col] += jac[18 * e + 6 * i + k] * res[3 * e + i];
          diag[col] += jac[18 * e + 6 * i + k] * jac[18 * e + 6 * i + k];
        }
  };
  auto grad_max = [&]() {
    double mx = 0;
    for (int j = 0; j < N; ++j) mx = std::max(mx, std::fabs(g[j] / scale[j]));
    return mx;
  };
  double cost = P.cost(aa);
  S.lm_initial_cost = cost;
  S.lm_iterations = 0;
  S.lm_successful_steps = 0;
  S.lm_termination = 0;
  double radius = lm.initial_radius, decrease_factor = 2.0;
  evaluate();
  bool stop = grad_max() <= lm.gradient_tolerance;
  if (stop) S.lm_termination = 2;
  std::vector<double> A;
  for (uint32_t iter = 1; !stop && iter <= lm.max_iterations; ++iter) {
    S.lm_iterations = iter;
    std::vector<double> D2(N);
    for (int j = 0; j < N; ++j) D2[j] = std::min(std::max(diag[j], 1e-6), 1e32) / radius;
    A.assign((size_t)N * N, 0.0);
    for (size_t e = 0; e < ne; ++e)
      for (int k = 0; k < 6; ++k)
        for (int l = 0; l < 6; ++l) {
          const size_t ck = 3 * (size_t)ab[2 * e + (k / 3)] + k % 3, cl = 3 * (size_t)ab[2 * e + (l / 3)] + l % 3;
          double s = 0.0;
          for (int i = 0; i < 3; ++i) s += jac[18 * e + 6 * i + k] * jac[18 * e + 6 * i + l];
          A[ck * N + cl] += s;
        }
    for (int j = 0; j < N; ++j) A[(size_t)j * N + j] += D2[j];
    for (int j = 0; j < N; ++j) delta[j] = -g[j];
    const bool pd = cholesky(A, N, n_threads);
    bool accepted = false;
    if (pd) {
      chol_solve(A, N, delta.data(), 1);
      double acc = 0.0;
      for (int j = 0; j < N; ++j) acc += delta[j] * (D2[j] * delta[j] - g[j]);
      const double model_cost_change = 0.5 * acc;
      if (model_cost_change > 0.0 && std::isfinite(model_cost_change)) {
        double dn = 0.0, xn = 0.0;
        for (int j = 0; j < N; ++j) {
          const double d = delta[j] * scale[j];
          aa_new[j] = aa[j] + d;
          dn += d * d;
          xn += aa[j] * aa[j];
        }
        if (std::sqrt(dn) <= lm.parameter_tolerance * (std::sqrt(xn) + lm.parameter_tolerance)) {
          S.lm_termination = 3;
          break;
        }
        const double new_cost = P.cost(aa_new);
        const double relative_decrease = (cost - new_cost) / model_cost_change;
        if (relative_decrease > 1e-3) {
          accepted = true;
          aa.swap(aa_new);
          const double cost_change = cost - new_cost;
          const double t = 2.0 * relative_decrease - 1.0;
          radius = radius / std::max(1.0 / 3.0, 1.0 - t * t * t);
          radius = std::min(1e16, radius);
          decrease_factor = 2.0;
          S.lm_successful_steps++;
          const bool ftol = std::fabs(cost_change) < lm.function_tolerance * cost;
          cost = new_cost;
          evaluate();
          if (ftol) { S.lm_termination = 1; break; }
          if (grad_max() <= lm.gradient_tolerance) { S.lm_termination = 2; break; }
        }
      }
    }
    if (!accepted) {
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      if (radius < 1e-32) { S.lm_termination = 4; break; }
    }
  }
  S.lm_final_cost = cost;
  for (uint32_t a = 0; a < m; ++a) rp::angle_axis_to_rotation(&aa[3 * (size_t)a], &Rl[9 * (size_t)a]);
  apply_gauge(Rl, m);
  return 0;
}

}  // namespace ra
}  // namespace orc

using namespace orc::ra;

extern "C" {

float orc_rotavg_cycle_error(const double* Rij, const double* Rjk, const double* Rik) { return cycle_error_deg(Rij, Rjk, Rik); }

int64_t orc_rotavg_triplets(const uint32_t* ij, const double* R, uint64_t E, uint32_t n_views, float thr, uint32_t* tri, float* err,
                            uint8_t* valid, uint64_t cap) {
  // edge lookup by (i < j); R is R_ij of the canonical orientation
  std::vector<std::vector<std::pair<uint32_t, uint64_t>>> up(n_views);
  for (uint64_t e = 0; e < E; ++e) up[std::min(ij[2 * e], ij[2 * e + 1])].push_back({std::max(ij[2 * e], ij[2 * e + 1]), e});
  for (auto& u : up) std::sort(u.begin(), u.end());
  auto find = [&](uint32_t a, uint32_t b) -> int64_t {
    const auto& u = up[a];
    auto it = std::lower_bound(u.begin(), u.end(), std::make_pair(b, (uint64_t)0));
    return (it != u.end() && it->first == b) ? (int64_t)it->second : -1;
  };
  uint64_t n = 0;
  for (uint32_t i = 0; i < n_views; ++i)
    for (const auto& pj : up[i])
      for (const auto& pk : up[pj.first]) {
        const int64_t eik = find(i, pk.first);
        if (eik < 0) continue;
        if (n < cap) {
          tri[3 * n] = i; tri[3 * n + 1] = pj.first; tri[3 * n + 2] = pk.first;
          err[n] = cycle_error_deg(R + 9 * pj.second, R + 9 * pk.second, R + 9 * (uint64_t)eik);
          valid[n] = err[n] < thr;
        }
        ++n;
      }
  return (int64_t)n;
}

int orc_largest_biedge_component(const uint32_t* ij, uint64_t E, uint32_t n_views, uint8_t* kept) {
  std::vector<uint32_t> eu(E), ev(E);
  for (uint64_t e = 0; e < E; ++e) { eu[e] = ij[2 * e]; ev[e] = ij[2 * e + 1]; }
  std::vector<int> comp;
  const int best = largest_biedge_component(n_views, eu, ev, comp);
  int cnt = 0;
  for (uint32_t v = 0; v < n_views; ++v) {
    kept[v] = best >= 0 && comp[v] == best;
    cnt += kept[v];
  }
  return cnt;
}

uint32_t orc_rotavg_l2_subspace(const uint32_t* ab, const double* R, uint64_t E, uint32_t m, double* M, double* Q, int n_threads) {
  const std::vector<uint32_t> vab(ab, ab + 2 * E);
  const std::vector<double> vR(R, R + 9 * E);
  if (M) {
    std::vector<double> Mv;
    assemble_M(vab, vR, m, Mv, nullptr);
    std::memcpy(M, Mv.data(), Mv.size() * sizeof(double));
  }
  std::vector<double> Qv;
  const uint32_t it = l2_subspace(vab, vR, m, Qv, n_threads > 0 ? n_threads : omp_get_max_threads());
  if (it) std::memcpy(Q, Qv.data(), Qv.size() * sizeof(double));
  return it;
}

int orc_rotation_averaging(const orc_relpose_result* rel, uint64_t n_rel, uint32_t n_views, const orc_rotavg_options* o, double* rotations,
                           uint8_t* view_kept, uint8_t* edge_kept, uint32_t* edge_support, orc_rotavg_summary* S, int n_threads) {
  if (n_threads <= 0) n_threads = omp_get_max_threads();
  std::memset(S, 0, sizeof(*S));
  S->lm_termination = -1;
  if (o->method == 1) return -5;
  if (o->method != 0 || !(o->max_angular_error_deg > 0.0)) return -1;
  std::memset(rotations, 0, (size_t)n_views * 9 * sizeof(double));
  std::memset(view_kept, 0, n_views);
  if (edge_kept) std::memset(edge_kept, 0, n_rel);
  if (edge_support) std::memset(edge_support, 0, n_rel * sizeof(uint32_t));
  // ---- edges ----
  std::vector<uint64_t> src;
  std::vector<uint32_t> ij;
  std::vector<double> R;
  for (uint64_t k = 0; k < n_rel; ++k) {
    const orc_relpose_result& r = rel[k];
    if (r.status != ORC_RELPOSE_OK) continue;
    if (r.I == r.J || r.I >= n_views || r.J >= n_views) return -1;
    src.push_back(k);
    ij.push_back(std::min(r.I, r.J));
    ij.push_back(std::max(r.I, r.J));
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) R.push_back(r.I < r.J ? r.rotation[3 * a + b] : r.rotation[3 * b + a]);
  }
  const uint64_t E = src.size();
  S->n_edges = E;
  {
    std::vector<std::pair<uint32_t, uint32_t>> pr(E);
    for (uint64_t e = 0; e < E; ++e) pr[e] = {ij[2 * e], ij[2 * e + 1]};
    std::sort(pr.begin(), pr.end());
    for (size_t e = 1; e < pr.size(); ++e)
      if (pr[e] == pr[e - 1]) return -1;
  }
  // ---- triplets: every i < j < k, its own loop ----
  std::vector<std::vector<std::pair<uint32_t, uint64_t>>> up(n_views);
  for (uint64_t e = 0; e < E; ++e) up[ij[2 * e]].push_back({ij[2 * e + 1], e});
  for (auto& u : up) std::sort(u.begin(), u.end());
  std::vector<uint32_t> support(E, 0);
  const float thr = (float)o->max_angular_error_deg;
  uint64_t nt = 0, nv = 0;
#pragma omp parallel num_threads(n_threads) reduction(+ : nt, nv)
  {
    std::vector<int64_t> slot(n_views, -1);
    std::vector<uint32_t> sup(E, 0);
#pragma omp for schedule(dynamic, 1)
    for (int64_t i = 0; i < (int64_t)n_views; ++i) {
      for (const auto& p : up[(size_t)i]) slot[p.first] = (int64_t)p.second;
      for (const auto& pj : up[(size_t)i])
        for (const auto& pk : up[pj.first]) {
          const int64_t eik = slot[pk.first];
          if (eik < 0) continue;
          ++nt;
          if (cycle_error_deg(&R[9 * pj.second], &R[9 * pk.second], &R[9 * (size_t)eik]) < thr) {
            ++nv;
            sup[pj.second]++;
            sup[pk.second]++;
            sup[(size_t)eik]++;
          }
        }
      for (const auto& p : up[(size_t)i]) slot[p.first] = -1;
    }
#pragma omp critical
    for (uint64_t e = 0; e < E; ++e) support[e] += sup[e];
  }
  S->n_triplets = nt;
  S->n_valid_triplets = nv;
  if (edge_support)
    for (uint64_t e = 0; e < E; ++e) edge_support[src[e]] = support[e];
  // ---- the largest bi-edge-connected component of the supported edges ----
  std::vector<uint32_t> eu, ev;
  std::vector<uint64_t> eid;
  for (uint64_t e = 0; e < E; ++e)
    if (support[e]) { eu.push_back(ij[2 * e]); ev.push_back(ij[2 * e + 1]); eid.push_back(e); }
  std::vector<int> comp;
  const int best = largest_biedge_component(n_views, eu, ev, comp);
  if (best < 0) return 0;
  std::vector<uint32_t> local(n_views, UINT32_MAX), kview;
  for (uint32_t v = 0; v < n_views; ++v)
    if (comp[v] == best) { local[v] = (uint32_t)kview.size(); kview.push_back(v); }
  const uint32_t m = (uint32_t)kview.size();
  if (m > 4096) return -5;
  // kept edges in (a, b) order
  std::vector<std::pair<std::pair<uint32_t, uint32_t>, uint64_t>> ke;
  for (size_t q = 0; q < eid.size(); ++q)
    if (local[eu[q]] != UINT32_MAX && local[ev[q]] != UINT32_MAX) ke.push_back({{local[eu[q]], local[ev[q]]}, eid[q]});
  std::sort(ke.begin(), ke.end());
  std::vector<uint32_t> ab;
  std::vector<double> kR;
  for (const auto& k : ke) {
    ab.push_back(k.first.first);
    ab.push_back(k.first.second);
    kR.insert(kR.end(), &R[9 * k.second], &R[9 * k.second] + 9);
    if (edge_kept) edge_kept[src[k.second]] = 1;
  }
  S->success = 1;
  S->n_kept_views = m;
  S->n_kept_edges = ke.size();
  for (uint32_t v : kview) view_kept[v] = 1;
  std::vector<double> Rl;
  if (run_l2(ab, kR, m, *o, Rl, *S, n_threads)) return -2;
  for (uint32_t a = 0; a < m; ++a) std::memcpy(rotations + 9 * (size_t)kview[a], &Rl[9 * (size_t)a], 9 * sizeof(double));
  return 0;
}

}  // extern "C"
