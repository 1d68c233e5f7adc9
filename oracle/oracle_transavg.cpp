// oracle_transavg.cpp -- CPU ORACLE (test infrastructure; see oracle_transavg.h), liboracle_transavg.so (oracle/transavg.mk).
//
// Restates GlobalSfM_Translation_AveragingSolver's Translation_averaging for TRANSLATION_AVERAGING_L2_DISTANCE_CHORDAL
// and TRANSLATION_AVERAGING_SOFTL1, the third step of the global pipeline (GlobalSfMReconstructionEngine_RelativeMotions::
// Compute_Global_Translations, reached from src/threads/R3DTriangulationThread.cpp:201-250; un-vendored OpenMVG 1.4,
// SURVEY.md A.11), on the pairwise relative translations (DESIGN.md sec. 2):
//   * edges: OK relative poses with edge_use set and both views rotation-kept; CleanGraph_KeepLargestBiEdge_Nodes +
//     KeepOnlyReferencedElement (oracle_rotavg.cpp's Tarjan), reindexing in view id order;
//   * L2 chordal (solve_translations_problem_l2_chordal, 1DSfM): centres C, one ChordFunctor residual per edge
//     (C_J - C_I) / |C_J - C_I| - u, u = -R_J^T t_IJ / |t_IJ|, no loss, start from a splitmix64 draw in [0, 1);
//   * soft-L1 (solve_translations_problem_softl1): translations t (start 1) and one scale s >= 1 per edge (start 1),
//     RelativeTranslationError t_J - AngleAxisRotatePoint(aa(R_J R_I^T), t_I) - s t_IJ / |t_IJ|, SoftLOneLoss with the
//     Corrector's sqrt(rho') scaling;
//   * the trust-region LM of oracle_ba.cpp (SURVEY.md A.7) with Jacobians from forward-mode jets, the scales
//     eliminated from the dense normal equations by their 1 x 1 Schur complements; bounds as Ceres: Plus clamps s to
//     >= 1, the step norm is taken on the clamped step, the gradient tolerance uses |x - Plus(x, -g)|, the model cost
//     change the unclamped step; in addition a scale on its bound whose gradient points out of the box is held for the
//     step (DESIGN.md sec. 2: without it the clamped steps stall).  Gauge: the lowest kept view has C = 0 / t = 0 exactly and is held.
// PARITY UNPINNED.
#include "oracle_transavg.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>
#include <omp.h>

namespace orc {
namespace rp {  // oracle_relpose.cpp (liboracle_relpose.so)
void rotation_to_angle_axis(const double* R, double* aa);
}  // namespace rp
namespace ra {  // oracle_rotavg.cpp (liboracle_rotavg.so)
int largest_biedge_component(uint32_t n, const std::vector<uint32_t>& eu, const std::vector<uint32_t>& ev, std::vector<int>& comp);
bool cholesky(std::vector<double>& A, int n, int n_threads);
void chol_solve(const std::vector<double>& L, int n, double* b, int k);
}  // namespace ra

namespace ta {

const int kChordal = 2, kSoftL1 = 3;

struct Jet {
  double a;
  double v[7];
};
Jet jc(double x) { Jet r; r.a = x; for (int i = 0; i < 7; ++i) r.v[i] = 0.0; return r; }
Jet operator+(const Jet& x, const Jet& y) { Jet r; r.a = x.a + y.a; for (int i = 0; i < 7; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
Jet operator-(const Jet& x, const Jet& y) { Jet r; r.a = x.a - y.a; for (int i = 0; i < 7; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
Jet operator*(const Jet& x, const Jet& y) { Jet r; r.a = x.a * y.a; for (int i = 0; i < 7; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
Jet operator/(const Jet& x, const Jet& y) { Jet r; const double inv = 1.0 / y.a; r.a = x.a * inv; for (int i = 0; i < 7; ++i) r.v[i] = (x.v[i] - r.a * y.v[i]) * inv; return r; }
Jet operator-(const Jet& x, double s) { Jet r = x; r.a -= s; return r; }
Jet operator*(const Jet& x, double s) { Jet r; r.a = x.a * s; for (int i = 0; i < 7; ++i) r.v[i] = x.v[i] * s; return r; }
Jet sqrt(const Jet& x) { Jet r; r.a = std::sqrt(x.a); const double d = 0.5 / r.a; for (int i = 0; i < 7; ++i) r.v[i] = x.v[i] * d; return r; }
double sqrt(double x) { return std::sqrt(x); }

template <class T>
void chordal_residual(const T* xi, const T* xj, const double* u, T* r) {  // ChordFunctor, weight 1
  const T d0 = xj[0] - xi[0], d1 = xj[1] - xi[1], d2 = xj[2] - xi[2];
  const T nrm = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  r[0] = d0 / nrm - u[0];
  r[1] = d1 / nrm - u[1];
  r[2] = d2 / nrm - u[2];
}
template <class T>
void softl1_residual(const T* ti, const T* tj, const T& s, const double* e, T* r) {  // RelativeTranslationError
  const double* aa = e;
  const double* u = e + 3;
  T p[3];  // ceres::AngleAxisRotatePoint(aa, t_i)
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > std::numeric_limits<double>::epsilon()) {
    const double th = std::sqrt(th2);
    const double c = std::cos(th), sn = std::sin(th), inv = 1.0 / th;
    const double w[3] = {aa[0] * inv, aa[1] * inv, aa[2] * inv};
    const T wx[3] = {ti[2] * w[1] - ti[1] * w[2], ti[0] * w[2] - ti[2] * w[0], ti[1] * w[0] - ti[0] * w[1]};
    const T tmp = (ti[0] * w[0] + ti[1] * w[1] + ti[2] * w[2]) * (1.0 - c);
    for (int k = 0; k < 3; ++k) p[k] = ti[k] * c + wx[k] * sn + tmp * w[k];
  } else {
    const T wx[3] = {ti[2] * aa[1] - ti[1] * aa[2], ti[0] * aa[2] - ti[2] * aa[0], ti[1] * aa[0] - ti[0] * aa[1]};
    for (int k = 0; k < 3; ++k) p[k] = ti[k] + wx[k];
  }
  for (int k = 0; k < 3; ++k) r[k] = (tj[k] - p[k]) - s * u[k];
}

double softl1_rho(double sq, double a, double* rho1) {  // ceres::SoftLOneLoss
  const double b = a * a, c = 1.0 / b;
  const double sum = 1.0 + sq * c;
  const double tmp = std::sqrt(sum);
  *rho1 = std::max(std::numeric_limits<double>::min(), 1.0 / tmp);
  return 2.0 * b * (tmp - 1.0);
}

double start_value(uint64_t k) {  // the device's chordal start (transavg.cu)
  uint64_t z = k * 0x9E3779B97F4A7C15ull + 0x6A09E667F3BCC909ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

// the raw residual and Jacobian of one edge at view coordinates xi, xj and scale s
void edge_jet(int method, const double* xi, const double* xj, double s, const double* e, double* res, double* jac) {
  Jet a[3], b[3], r[3];
  for (int k = 0; k < 3; ++k) {
    a[k] = jc(xi[k]);
    a[k].v[k] = 1.0;
    b[k] = jc(xj[k]);
    b[k].v[3 + k] = 1.0;
  }
  if (method == kChordal) {
    chordal_residual(a, b, e, r);
  } else {
    Jet sj = jc(s);
    sj.v[6] = 1.0;
    softl1_residual(a, b, sj, e, r);
  }
  for (int i = 0; i < 3; ++i) {
    res[i] = r[i].a;
    for (int k = 0; k < 7; ++k) jac[7 * i + k] = r[i].v[k];
  }
}

struct Problem {
  int method;
  std::vector<uint32_t> ab;  // 2 per kept edge: local (I, J) in the record's orientation
  std::vector<double> ed;    // 6 per kept edge
  uint32_t m;
  double loss;
  int n_threads;
  size_t ne() const { return ab.size() / 2; }
  int N() const { return 3 * ((int)m - 1); }
  void coords(const std::vector<double>& x, uint32_t v, double* p) const {
    for (int k = 0; k < 3; ++k) p[k] = v == 0 ? 0.0 : x[3 * (size_t)(v - 1) + k];
  }
  double cost(const std::vector<double>& x) const {
    std::vector<double> c(ne());
#pragma omp parallel for schedule(static) num_threads(n_threads)
    for (int64_t e = 0; e < (int64_t)ne(); ++e) {
      double xi[3], xj[3], r[3];
      coords(x, ab[2 * e], xi);
      coords(x, ab[2 * e + 1], xj);
      if (method == kChordal) {
        chordal_residual(xi, xj, &ed[6 * (size_t)e], r);
        c[(size_t)e] = 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
      } else {
        softl1_residual(xi, xj, x[(size_t)N() + (size_t)e], &ed[6 * (size_t)e], r);
        double rho1;
        c[(size_t)e] = 0.5 * softl1_rho(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], loss, &rho1);
      }
    }
    double s = 0.0;
    for (double v : c) s += v;
    return s;
  }
};

// LM on x (free view coordinates, then the scales), oracle_ba.cpp's state machine with the bounds s >= 1
void run_lm(const Problem& P, std::vector<double>& x, uint32_t max_iterations, double function_tolerance, const orc_ba_options& lm,
            orc_transavg_summary& S) {
  const bool softl1 = P.method == kSoftL1;
  const size_t ne = P.ne();
  const int N = P.N();
  const size_t Nv = x.size();
  std::vector<double> res(3 * ne), jac(21 * ne), scale(Nv, 1.0), g(Nv), diag(Nv), delta(Nv), x_new(Nv);
  // column of entry k (0..6) of edge e, -1 for the held view
  auto column = [&](size_t e, int k) -> int64_t {
    if (k == 6) return (int64_t)N + (int64_t)e;
    const uint32_t v = P.ab[2 * e + (k / 3)];
    return v == 0 ? -1 : 3 * (int64_t)(v - 1) + k % 3;
  };
  bool have_scale = false;
  auto evaluate = [&]() {
#pragma omp parallel for schedule(static) num_threads(P.n_threads)
    for (int64_t e = 0; e < (int64_t)ne; ++e) {
      double xi[3], xj[3];
      P.coords(x, P.ab[2 * e], xi);
      P.coords(x, P.ab[2 * e + 1], xj);
      double* r = &res[3 * (size_t)e];
      double* J = &jac[21 * (size_t)e];
      edge_jet(P.method, xi, xj, softl1 ? x[(size_t)N + (size_t)e] : 0.0, &P.ed[6 * (size_t)e], r, J);
      if (softl1) {
        double rho1;
        softl1_rho(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], P.loss, &rho1);
        const double sq = std::sqrt(rho1);
        for (int i = 0; i < 3; ++i) r[i] *= sq;
        for (int k = 0; k < 21; ++k) J[k] *= sq;
      }
    }
    const int nk = softl1 ? 7 : 6;
    if (!have_scale) {
      std::vector<double> n2(Nv, 0.0);
      for (size_t e = 0; e < ne; ++e)
        for (int k = 0; k < nk; ++k) {
          const int64_t c = column(e, k);
          if (c < 0) continue;
          for (int i = 0; i < 3; ++i) n2[(size_t)c] += jac[21 * e + 7 * i + k] * jac[21 * e + 7 * i + k];
        }
      for (size_t j = 0; j < Nv; ++j) scale[j] = 1.0 / (1.0 + std::sqrt(n2[j]));
      have_scale = true;
    }
    for (size_t e = 0; e < ne; ++e)
      for (int k = 0; k < 7; ++k) {
        const int64_t c = k < nk ? column(e, k) : -1;
        for (int i = 0; i < 3; ++i) jac[21 * e + 7 * i + k] = c < 0 ? 0.0 : jac[21 * e + 7 * i + k] * scale[(size_t)c];
      }
    std::fill(g.begin(), g.end(), 0.0);
    std::fill(diag.begin(), diag.end(), 0.0);
    for (size_t e = 0; e < ne; ++e)
      for (int k = 0; k < nk; ++k) {
        const int64_t c = column(e, k);
        if (c < 0) continue;
        for (int i = 0; i < 3; ++i) {
          g[(size_t)c] += jac[21 * e + 7 * i + k] * res[3 * e + i];
          diag[(size_t)c] += jac[21 * e + 7 * i + k] * jac[21 * e + 7 * i + k];
        }
      }
  };
  auto grad_max = [&]() {  // |x - Plus(x, -g)|_inf on the unscaled gradient
    double mx = 0;
    for (size_t j = 0; j < Nv; ++j) {
      const double gt = g[j] / scale[j];
      mx = std::max(mx, std::fabs((int)j < N ? gt : x[j] - std::max(x[j] - gt, 1.0)));
    }
    return mx;
  };
  double cost = P.cost(x);
  S.lm_initial_cost = cost;
  S.lm_iterations = 0;
  S.lm_successful_steps = 0;
  S.lm_termination = 0;
  double radius = lm.initial_radius, decrease_factor = 2.0;
  evaluate();
  bool stop = grad_max() <= lm.gradient_tolerance;
  if (stop) S.lm_termination = 2;
  std::vector<double> A;
  std::vector<double> js(3 * ne), V(ne), wv(6 * ne);
  for (uint32_t iter = 1; !stop && iter <= max_iterations; ++iter) {
    S.lm_iterations = iter;
    std::vector<double> D2(Nv);
    for (size_t j = 0; j < Nv; ++j) D2[j] = std::min(std::max(diag[j], 1e-6), 1e32) / radius;
    // reduced normal equations: J_t^T J_t + D_t^2 - sum_e w w^T / V_e, right-hand side -g_t + sum_e w g_s / V_e
    A.assign((size_t)N * N, 0.0);
    std::vector<double> rhs(N, 0.0);
    // scales on their bound whose gradient pushes them below it are held for this step (an active set)
    std::vector<char> held(ne, 0);
    for (size_t e = 0; e < ne && softl1; ++e) held[e] = x[(size_t)N + e] <= 1.0 && g[(size_t)N + e] > 0.0;
    for (size_t e = 0; e < ne; ++e) {
      const double* J = &jac[21 * e];
      const bool elim = softl1 && !held[e];
      if (elim) {
        for (int i = 0; i < 3; ++i) js[3 * e + i] = J[7 * i + 6];
        const double ds = js[3 * e] * js[3 * e] + js[3 * e + 1] * js[3 * e + 1] + js[3 * e + 2] * js[3 * e + 2];
        V[e] = ds + std::min(std::max(ds, 1e-6), 1e32) / radius;
        for (int k = 0; k < 6; ++k) wv[6 * e + k] = J[k] * js[3 * e] + J[7 + k] * js[3 * e + 1] + J[14 + k] * js[3 * e + 2];
      }
      for (int p = 0; p < 2; ++p) {
        const int64_t cp = column(e, 3 * p);
        if (cp < 0) continue;
        for (int q = 0; q < 2; ++q) {
          const int64_t cq = column(e, 3 * q);
          if (cq < 0) continue;
          for (int k = 0; k < 3; ++k)
            for (int l = 0; l < 3; ++l) {
              double s = (J[3 * p + k] * J[3 * q + l] + J[7 + 3 * p + k] * J[7 + 3 * q + l]) + J[14 + 3 * p + k] * J[14 + 3 * q + l];
              if (elim) s = s - wv[6 * e + 3 * p + k] * wv[6 * e + 3 * q + l] / V[e];
              A[(size_t)(cp + k) * N + (size_t)(cq + l)] += s;
            }
        }
        if (elim)
          for (int k = 0; k < 3; ++k) rhs[(size_t)(cp + k)] = rhs[(size_t)(cp + k)] + wv[6 * e + 3 * p + k] * g[(size_t)N + e] / V[e];
      }
    }
    for (int j = 0; j < N; ++j) {
      A[(size_t)j * N + j] += D2[j];
      delta[j] = rhs[j] - g[j];
    }
    const bool pd = ra::cholesky(A, N, P.n_threads);
    bool accepted = false;
    if (pd) {
      ra::chol_solve(A, N, delta.data(), 1);
      for (size_t e = 0; e < ne && softl1; ++e) {  // the scale steps
        if (held[e]) {
          delta[(size_t)N + e] = 0.0;
          continue;
        }
        double acc = g[(size_t)N + e];
        for (int p = 0; p < 2; ++p) {
          const int64_t cp = column(e, 3 * p);
          if (cp < 0) continue;
          for (int k = 0; k < 3; ++k) acc = acc + wv[6 * e + 3 * p + k] * delta[(size_t)(cp + k)];
        }
        delta[(size_t)N + e] = -acc / V[e];
      }
      double acc = 0.0;
      for (size_t j = 0; j < Nv; ++j) acc += delta[j] * (D2[j] * delta[j] - g[j]);
      const double model_cost_change = 0.5 * acc;
      if (model_cost_change > 0.0 && std::isfinite(model_cost_change)) {
        double dn = 0.0, xn = 0.0;
        for (size_t j = 0; j < Nv; ++j) {
          const double d = delta[j] * scale[j];
          if ((int)j < N) {
            x_new[j] = x[j] + d;
            dn += d * d;
          } else {
            x_new[j] = std::max(x[j] + d, 1.0);
            dn += (x_new[j] - x[j]) * (x_new[j] - x[j]);
          }
          xn += x[j] * x[j];
        }
        if (std::sqrt(dn) <= lm.parameter_tolerance * (std::sqrt(xn) + lm.parameter_tolerance)) {
          S.lm_termination = 3;
          break;
        }
        const double new_cost = P.cost(x_new);
        const double relative_decrease = (cost - new_cost) / model_cost_change;
        if (relative_decrease > 1e-3) {
          accepted = true;
          x.swap(x_new);
          const double cost_change = cost - new_cost;
          const double t = 2.0 * relative_decrease - 1.0;
          radius = radius / std::max(1.0 / 3.0, 1.0 - t * t * t);
          radius = std::min(1e16, radius);
          decrease_factor = 2.0;
          S.lm_successful_steps++;
          const bool ftol = std::fabs(cost_change) < function_tolerance * cost;
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
}

}  // namespace ta
}  // namespace orc

using namespace orc::ta;

extern "C" {

void orc_transavg_edge(int method, const double* xi, const double* xj, double s, const double* edata, double* res, double* jac) {
  edge_jet(method, xi, xj, s, edata, res, jac);
}

double orc_softl1_rho(double sq, double a, double* rho1) { return softl1_rho(sq, a, rho1); }

int orc_translation_averaging(const orc_relpose_result* rel, uint64_t n_rel, const uint8_t* edge_use, const double* rot,
                              const uint8_t* rot_kept, uint32_t n_views, const orc_transavg_options* o, double* centers,
                              double* translations, uint8_t* view_kept, uint8_t* edge_kept, orc_transavg_summary* S, int n_threads) {
  const auto t0 = std::chrono::steady_clock::now();
  if (n_threads <= 0) n_threads = omp_get_max_threads();
  std::memset(S, 0, sizeof(*S));
  S->lm_termination = -1;
  if (o->method == 1) return -5;
  if ((o->method != kChordal && o->method != kSoftL1) || (o->method == kSoftL1 && !(o->softl1_loss > 0.0))) return -1;
  std::memset(centers, 0, (size_t)n_views * 3 * sizeof(double));
  std::memset(translations, 0, (size_t)n_views * 3 * sizeof(double));
  std::memset(view_kept, 0, n_views);
  if (edge_kept) std::memset(edge_kept, 0, n_rel);
  // ---- edges ----
  std::vector<std::pair<std::pair<uint32_t, uint32_t>, uint64_t>> cand;  // ((min, max), record)
  for (uint64_t k = 0; k < n_rel; ++k) {
    const orc_relpose_result& r = rel[k];
    if (r.status != ORC_RELPOSE_OK || (edge_use && !edge_use[k])) continue;
    if (r.I == r.J || r.I >= n_views || r.J >= n_views) return -1;
    const double tn = r.translation[0] * r.translation[0] + r.translation[1] * r.translation[1] + r.translation[2] * r.translation[2];
    if (!std::isfinite(tn) || !(tn > 0.0)) return -1;
    cand.push_back({{std::min(r.I, r.J), std::max(r.I, r.J)}, k});
  }
  std::sort(cand.begin(), cand.end());
  for (size_t k = 1; k < cand.size(); ++k)
    if (cand[k].first == cand[k - 1].first) return -1;
  std::vector<uint32_t> eu, ev;
  std::vector<uint64_t> src;
  for (const auto& c : cand)
    if (rot_kept[c.first.first] && rot_kept[c.first.second]) {
      eu.push_back(c.first.first);
      ev.push_back(c.first.second);
      src.push_back(c.second);
    }
  S->n_edges = src.size();
  std::vector<int> comp;
  const int best = orc::ra::largest_biedge_component(n_views, eu, ev, comp);
  if (best < 0) return 0;
  std::vector<uint32_t> local(n_views, UINT32_MAX), kview;
  for (uint32_t v = 0; v < n_views; ++v)
    if (comp[v] == best) { local[v] = (uint32_t)kview.size(); kview.push_back(v); }
  const uint32_t m = (uint32_t)kview.size();
  if (m > 4096) return -5;
  Problem P{o->method, {}, {}, m, o->softl1_loss, n_threads};
  const bool softl1 = o->method == kSoftL1;
  for (size_t q = 0; q < src.size(); ++q) {
    if (local[eu[q]] == UINT32_MAX || local[ev[q]] == UINT32_MAX) continue;
    const orc_relpose_result& r = rel[src[q]];
    P.ab.push_back(local[r.I]);
    P.ab.push_back(local[r.J]);
    const double* t = r.translation;
    const double tn = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    const double u[3] = {t[0] / tn, t[1] / tn, t[2] / tn};
    const double* RI = rot + 9 * (size_t)r.I;
    const double* RJ = rot + 9 * (size_t)r.J;
    double e6[6] = {0, 0, 0, 0, 0, 0};
    if (!softl1) {
      for (int k = 0; k < 3; ++k) e6[k] = -(RJ[k] * u[0] + RJ[3 + k] * u[1] + RJ[6 + k] * u[2]);
    } else {
      double Rij[9];  // R_J R_I^T
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) Rij[3 * a + b] = RJ[3 * a] * RI[3 * b] + RJ[3 * a + 1] * RI[3 * b + 1] + RJ[3 * a + 2] * RI[3 * b + 2];
      orc::rp::rotation_to_angle_axis(Rij, e6);
      for (int k = 0; k < 3; ++k) e6[3 + k] = u[k];
    }
    P.ed.insert(P.ed.end(), e6, e6 + 6);
    if (edge_kept) edge_kept[src[q]] = 1;
  }
  const size_t ne = P.ne();
  S->success = 1;
  S->n_kept_views = m;
  S->n_kept_edges = ne;
  for (uint32_t v : kview) view_kept[v] = 1;
  const int N = P.N();
  std::vector<double> x((size_t)N + (softl1 ? ne : 0));
  for (int j = 0; j < N; ++j) x[j] = softl1 ? 1.0 : start_value((uint64_t)j);
  for (size_t e = 0; softl1 && e < ne; ++e) x[(size_t)N + e] = 1.0;
  const uint32_t max_it = o->lm.max_iterations > 0 ? o->lm.max_iterations : (softl1 ? std::max<uint32_t>(50, 2 * (uint32_t)ne) : 500u);
  const double ftol = o->lm.function_tolerance > 0.0 ? o->lm.function_tolerance : (softl1 ? 1e-6 : 1e-7);
  run_lm(P, x, max_it, ftol, o->lm, *S);
  for (uint32_t a = 0; a < m; ++a) {
    const uint32_t v = kview[a];
    const double* R = rot + 9 * (size_t)v;
    double p[3];
    P.coords(x, a, p);
    double* C = centers + 3 * (size_t)v;
    double* t = translations + 3 * (size_t)v;
    for (int k = 0; k < 3; ++k) {
      if (softl1) {
        t[k] = p[k];
        C[k] = -(R[k] * p[0] + R[3 + k] * p[1] + R[6 + k] * p[2]);
      } else {
        C[k] = p[k];
        t[k] = -(R[3 * k] * p[0] + R[3 * k + 1] * p[1] + R[3 * k + 2] * p[2]);
      }
    }
  }
  S->ms_host = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}

}  // extern "C"
