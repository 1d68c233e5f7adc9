// transavg.cu -- global camera translations from the relative motions and the global rotations
// (r3d_translation_averaging).
// COMPILED WITH --fmad=false (regard3d_b200/build.py): residuals, Jacobians and the normal equations are written in the
// operation order of the CPU restatement (oracle/oracle_transavg.cpp), so both take the same LM path.
//
// Replaces GlobalSfM_Translation_AveragingSolver::Translation_averaging (OpenMVG 1.4, SURVEY.md A.11) for
// TRANSLATION_AVERAGING_L2_DISTANCE_CHORDAL and TRANSLATION_AVERAGING_SOFTL1, on the pairwise relative translations:
//   1. host (select_edges, shared with transavg_l1.cu): the usable edges, the largest bi-edge-connected component
//      (rotavg.cu's Tarjan), reindexing by view id.
//   2. Levenberg-Marquardt (averaging.cuh's loop around lm_trust_region.cuh's trust region), the lowest kept view held:
//      k_ta_eval (one thread per edge, forward-mode duals: residual, 3 x 7 Jacobian, soft-L1 corrector), k_ta_edge
//      (the scale columns' Jacobi scale and gradient), k_ta_system (one owner CTA per view block row: J^T J + D^2 with
//      each edge's scale eliminated in the same pass -- no floating-point atomics), k_chol_fused (ba.cu) on the 3(m-1)
//      reduced system, k_ta_back (the scale steps; a scale on its bound pushed outwards is held); the step clamps
//      s >= 1.  Fixed-order reductions: repeated calls are bit-identical.
#include "r3d_internal.cuh"
#include "averaging.cuh"
#include "relpose_math.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace r3d {
namespace ta {

constexpr int kChordal = 2;  // R3D_TRANSAVG_L2_CHORDAL
constexpr int kSoftL1 = 3;   // R3D_TRANSAVG_SOFTL1

// forward-mode dual: partials of (first view's 3 coordinates, second view's 3, the edge's scale)
using Dual = ra::Dual<7>;
using ra::sqrt;

// ChordFunctor (1DSfM): r = (x_J - x_I) / |x_J - x_I| - u, u = -R_J^T t_IJ / |t_IJ|
template <class T>
__device__ void chordal_residual(const T* xi, const T* xj, const double* u, T* r) {
  const T d0 = xj[0] - xi[0], d1 = xj[1] - xi[1], d2 = xj[2] - xi[2];
  const T nrm = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  r[0] = d0 / nrm - u[0];
  r[1] = d1 / nrm - u[1];
  r[2] = d2 / nrm - u[2];
}
// RelativeTranslationError: r = t_J - AngleAxisRotatePoint(aa_IJ, t_I) - s t_IJ / |t_IJ| (ceres::AngleAxisRotatePoint with
// a constant angle-axis)
template <class T>
__device__ void softl1_residual(const T* ti, const T* tj, const T& s, const double* e, T* r) {
  const double* aa = e;
  const double* u = e + 3;
  T p[3];
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > 2.220446049250313e-16) {
    const double th = ::sqrt(th2);
    const double c = ::cos(th), sn = ::sin(th), ti_ = 1.0 / th;
    const double w[3] = {aa[0] * ti_, aa[1] * ti_, aa[2] * ti_};
    const T wx[3] = {ti[2] * w[1] - ti[1] * w[2], ti[0] * w[2] - ti[2] * w[0], ti[1] * w[0] - ti[0] * w[1]};
    const T tmp = (ti[0] * w[0] + ti[1] * w[1] + ti[2] * w[2]) * (1.0 - c);
    for (int k = 0; k < 3; ++k) p[k] = ti[k] * c + wx[k] * sn + tmp * w[k];
  } else {
    const T wx[3] = {ti[2] * aa[1] - ti[1] * aa[2], ti[0] * aa[2] - ti[2] * aa[0], ti[1] * aa[0] - ti[0] * aa[1]};
    for (int k = 0; k < 3; ++k) p[k] = ti[k] + wx[k];
  }
  for (int k = 0; k < 3; ++k) r[k] = (tj[k] - p[k]) - s * u[k];
}

// ceres::SoftLOneLoss(a): rho(s) = 2 b (sqrt(1 + s / b) - 1), rho' = 1 / sqrt(1 + s / b), b = a^2
R3D_RP_HD double softl1_rho(double sq, double a, double* rho1) {
  const double b = a * a, c = 1.0 / b;
  const double sum = 1.0 + sq * c;
  const double tmp = ::sqrt(sum);
  *rho1 = fmax(2.2250738585072014e-308, 1.0 / tmp);
  return 2.0 * b * (tmp - 1.0);
}

__device__ __forceinline__ double view_coord(const double* x, uint32_t v, int k) { return v == 0 ? 0.0 : x[3 * (size_t)(v - 1) + k]; }

// per kept edge: the (corrector-scaled) residual (3) and Jacobian (3 x 7: first view, second view, scale)
template <int M>
__global__ void k_ta_eval(const double* __restrict__ x, const uint2* __restrict__ ab, const double* __restrict__ ed, uint32_t ne,
                          uint32_t N, double loss_a, double* __restrict__ res, double* __restrict__ jac) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  Dual xi[3], xj[3], r[3];
  for (int k = 0; k < 3; ++k) {
    xi[k] = ra::dconst<7>(view_coord(x, v.x, k));
    xi[k].v[k] = 1.0;
    xj[k] = ra::dconst<7>(view_coord(x, v.y, k));
    xj[k].v[3 + k] = 1.0;
  }
  double sq = 1.0;
  if (M == kChordal) {
    chordal_residual(xi, xj, ed + 6 * (size_t)e, r);
  } else {
    Dual s = ra::dconst<7>(x[N + e]);
    s.v[6] = 1.0;
    softl1_residual(xi, xj, s, ed + 6 * (size_t)e, r);
    double rho1;
    softl1_rho(r[0].a * r[0].a + r[1].a * r[1].a + r[2].a * r[2].a, loss_a, &rho1);
    sq = ::sqrt(rho1);  // Corrector, rho'' < 0 branch
  }
  for (int i = 0; i < 3; ++i) {
    res[3 * (size_t)e + i] = r[i].a * sq;
    for (int k = 0; k < 7; ++k) jac[21 * (size_t)e + 7 * i + k] = r[i].v[k] * sq;
  }
}

// per kept edge: 1/2 rho(|r|^2)
template <int M>
__global__ void k_ta_cost(const double* __restrict__ x, const uint2* __restrict__ ab, const double* __restrict__ ed, uint32_t ne,
                          uint32_t N, double loss_a, double* __restrict__ cost) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const uint2 v = ab[e];
  double xi[3], xj[3], r[3];
  for (int k = 0; k < 3; ++k) {
    xi[k] = view_coord(x, v.x, k);
    xj[k] = view_coord(x, v.y, k);
  }
  if (M == kChordal) {
    chordal_residual(xi, xj, ed + 6 * (size_t)e, r);
    cost[e] = 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
  } else {
    softl1_residual(xi, xj, x[N + e], ed + 6 * (size_t)e, r);
    double rho1;
    cost[e] = 0.5 * softl1_rho(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], loss_a, &rho1);
  }
}

// the scale column of edge e: mode 0 its Jacobi scale; mode 1 its gradient and diag(J^T J) (scaled)
__global__ void k_ta_edge(int mode, const double* __restrict__ res, const double* __restrict__ jac, uint32_t ne, uint32_t N,
                          double* __restrict__ scale, double* __restrict__ g, double* __restrict__ diag) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const double* J = jac + 21 * (size_t)e;
  if (mode == 0) {
    scale[N + e] = 1.0 / (1.0 + ::sqrt(J[6] * J[6] + J[13] * J[13] + J[20] * J[20]));
    return;
  }
  const double sc = scale[N + e];
  double gs = 0.0, ds = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double j = J[7 * i + 6] * sc;
    gs += j * res[3 * (size_t)e + i];
    ds += j * j;
  }
  g[N + e] = gs;
  diag[N + e] = ds;
}

// a scale on its bound whose gradient points out of the box is held for the step (an active set; DESIGN.md sec. 2)
__device__ __forceinline__ bool scale_held(const double* x, const double* g, uint32_t N, uint32_t e) {
  return x[N + e] <= 1.0 && g[N + e] > 0.0;
}

// the scaled Jacobian blocks of edge e seen from view a: Ja (its own 3 columns), Jb (the other view's), js (the scale)
// and, when the scale is eliminated, w_a = Ja^T js, w_b = Jb^T js and V = js^T js + D^2_s
struct EdgeBlocks {
  double Ja[9], Jb[9], js[3], wa[3], wb[3], V;
};
__device__ __forceinline__ void edge_blocks(const double* J, const double* scale, uint32_t N, uint32_t e, uint32_t a, uint32_t b,
                                            int oa, bool elim, double inv_radius, EdgeBlocks& B) {
  const int ob = 3 - oa;
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) {
      B.Ja[3 * i + k] = J[7 * i + oa + k] * scale[3 * (size_t)(a - 1) + k];
      B.Jb[3 * i + k] = b == 0 ? 0.0 : J[7 * i + ob + k] * scale[3 * (size_t)(b - 1) + k];
    }
  if (!elim) return;
  const double sc = scale[N + e];
  for (int i = 0; i < 3; ++i) B.js[i] = J[7 * i + 6] * sc;
  const double ds = B.js[0] * B.js[0] + B.js[1] * B.js[1] + B.js[2] * B.js[2];
  B.V = ds + fmin(fmax(ds, 1e-6), 1e32) * inv_radius;
  for (int k = 0; k < 3; ++k) {
    B.wa[k] = B.Ja[k] * B.js[0] + B.Ja[3 + k] * B.js[1] + B.Ja[6 + k] * B.js[2];
    B.wb[k] = B.Jb[k] * B.js[0] + B.Jb[3 + k] * B.js[1] + B.Jb[6 + k] * B.js[2];
  }
}

// Owner per free view a = blockIdx.x + 1 (reduced block row a - 1), its incident edges in neighbour order: its block row
// of the reduced system (J^T J + D^2, scaled before the block products, with every free scale eliminated) into the zeroed
// (N + 1) x N matrix and the reduced right-hand side into row N.  The held view 0 has no row or column.  Off-diagonal
// blocks first, one per incident edge to a free view.
__global__ void __launch_bounds__(128) k_ta_system(int softl1, const uint32_t* __restrict__ inc_ofs, const uint32_t* __restrict__ inc_nbr,
                                                   const uint32_t* __restrict__ inc_edge, const uint2* __restrict__ ab,
                                                   const double* __restrict__ jac, const double* __restrict__ x, uint32_t N,
                                                   const double* __restrict__ scale, const double* __restrict__ g,
                                                   const double* __restrict__ diag, double inv_radius, double* __restrict__ A) {
  const uint32_t a = blockIdx.x + 1, tid = threadIdx.x;
  const uint32_t ra_ = 3 * (a - 1);
  const uint32_t b0 = inc_ofs[a], b1 = inc_ofs[a + 1];
  auto col = [&](uint32_t e) -> int { return ab[e].x == a ? 0 : 3; };
  for (uint32_t p = b0 + tid; p < b1; p += blockDim.x) {
    const uint32_t e = inc_edge[p], b = inc_nbr[p];
    if (b == 0) continue;
    const bool elim = softl1 && !scale_held(x, g, N, e);
    EdgeBlocks B;
    edge_blocks(jac + 21 * (size_t)e, scale, N, e, a, b, col(e), elim, inv_radius, B);
    for (int k = 0; k < 3; ++k)
      for (int l = 0; l < 3; ++l) {
        double s = B.Ja[k] * B.Jb[l] + B.Ja[3 + k] * B.Jb[3 + l] + B.Ja[6 + k] * B.Jb[6 + l];
        if (elim) s = s - B.wa[k] * B.wb[l] / B.V;
        A[(size_t)(ra_ + k) * N + 3 * (b - 1) + l] = s;
      }
  }
  if (tid < 9) {  // diagonal block: sum over the incident edges in order, + D^2; the right-hand side
    const int k = (int)tid / 3, l = (int)tid % 3;
    double s = 0.0, q = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p], b = inc_nbr[p];
      const bool elim = softl1 && !scale_held(x, g, N, e);
      EdgeBlocks B;
      edge_blocks(jac + 21 * (size_t)e, scale, N, e, a, b, col(e), elim, inv_radius, B);
      double t = (B.Ja[k] * B.Ja[l] + B.Ja[3 + k] * B.Ja[3 + l]) + B.Ja[6 + k] * B.Ja[6 + l];
      if (elim) {
        t = t - B.wa[k] * B.wa[l] / B.V;
        q = q + B.wa[k] * g[N + e] / B.V;
      }
      s += t;
    }
    if (k == l) s += fmin(fmax(diag[ra_ + k], 1e-6), 1e32) * inv_radius;
    A[(size_t)(ra_ + k) * N + ra_ + l] = s;
    if (l == 0) A[(size_t)N * N + ra_ + k] = q - g[ra_ + k];
  }
}

// back-substitution of the scale steps: ds_e = -(g_s + w_a^T dt_a + w_b^T dt_b) / V_e (dt of the held view = 0), 0 for
// a held scale
__global__ void k_ta_back(const uint2* __restrict__ ab, const double* __restrict__ jac, const double* __restrict__ x,
                          const double* __restrict__ scale, const double* __restrict__ g, uint32_t ne, uint32_t N, double inv_radius,
                          double* __restrict__ delta) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  if (scale_held(x, g, N, e)) {
    delta[N + e] = 0.0;
    return;
  }
  const uint2 v = ab[e];
  const double* J = jac + 21 * (size_t)e;
  const double sc = scale[N + e];
  double js[3];
  for (int i = 0; i < 3; ++i) js[i] = J[7 * i + 6] * sc;
  const double ds = js[0] * js[0] + js[1] * js[1] + js[2] * js[2];
  const double V = ds + fmin(fmax(ds, 1e-6), 1e32) * inv_radius;
  double acc = g[N + e];
  for (int side = 0; side < 2; ++side) {
    const uint32_t u = side == 0 ? v.x : v.y;
    if (u == 0) continue;
    for (int k = 0; k < 3; ++k) {
      const double su = scale[3 * (size_t)(u - 1) + k];
      const double w = (J[3 * side + k] * su) * js[0] + (J[7 + 3 * side + k] * su) * js[1] + (J[14 + 3 * side + k] * su) * js[2];
      acc = acc + w * delta[3 * (size_t)(u - 1) + k];
    }
  }
  delta[N + e] = -acc / V;
}

// the chordal start (the oracle draws the same numbers): a splitmix64 stream of its own, uniform in [0, 1)
double start_value(uint64_t k) {
  uint64_t z = k * 0x9E3779B97F4A7C15ull + 0x6A09E667F3BCC909ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

int select_edges(r3d_ctx* ctx, const char* fn, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                 const double* rot, const uint8_t* rot_kept, uint32_t n_views, KeptEdges& K) {
  // edges: checked, canonical order (min, max); the record's orientation is kept
  struct Edge { uint32_t lo, hi; uint64_t src; };
  std::vector<Edge> edges;
  for (uint64_t k = 0; k < n_rel; ++k) {
    const r3d_relative_pose& r = rel[k];
    if (r.status != R3D_RELPOSE_OK || (edge_use && !edge_use[k])) continue;
    if (r.I == r.J) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "an edge joins a view to itself");
    if (r.I >= n_views || r.J >= n_views) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "view id >= n_views");
    const double* t = r.translation;
    const double tn = t[0] * t[0] + t[1] * t[1] + t[2] * t[2];
    if (!std::isfinite(tn) || !(tn > 0.0)) return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "a zero or non-finite translation");
    edges.push_back({std::min(r.I, r.J), std::max(r.I, r.J), k});
  }
  std::sort(edges.begin(), edges.end(), [](const Edge& a, const Edge& b) { return a.lo != b.lo ? a.lo < b.lo : a.hi < b.hi; });
  for (size_t k = 1; k < edges.size(); ++k)
    if (edges[k].lo == edges[k - 1].lo && edges[k].hi == edges[k - 1].hi)
      return fail(ctx, R3D_ERR_INVALID, std::string(fn) + "the same pair of views is given twice");
  edges.erase(std::remove_if(edges.begin(), edges.end(), [&](const Edge& e) { return !rot_kept[e.lo] || !rot_kept[e.hi]; }), edges.end());
  K.n_edges = edges.size();
  // the largest bi-edge-connected component, local ids in view id order
  std::vector<uint32_t> eu(edges.size()), ev(edges.size());
  for (size_t k = 0; k < edges.size(); ++k) { eu[k] = edges[k].lo; ev[k] = edges[k].hi; }
  std::vector<int> comp;
  const int best = ra::largest_biedge_component(n_views, eu, ev, comp);
  if (best < 0) return R3D_OK;
  std::vector<uint32_t> local(n_views, UINT32_MAX);
  for (uint32_t v = 0; v < n_views; ++v)
    if (comp[v] == best) { local[v] = (uint32_t)K.kview.size(); K.kview.push_back(v); }
  if (K.kview.size() > R3D_ROTAVG_MAX_VIEWS) {
    K.kview.clear();
    return fail(ctx, R3D_ERR_UNSUPPORTED, std::string(fn) + "more than R3D_ROTAVG_MAX_VIEWS views in the component");
  }
  for (const Edge& e : edges) {
    if (local[e.lo] == UINT32_MAX || local[e.hi] == UINT32_MAX) continue;
    const r3d_relative_pose& r = rel[e.src];
    K.kab.push_back(make_uint2(local[e.lo], local[e.hi]));
    K.ab.push_back(make_uint2(local[r.I], local[r.J]));
    K.src.push_back(e.src);
    const double* t = r.translation;
    const double tn = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    const double u[3] = {t[0] / tn, t[1] / tn, t[2] / tn};
    const double* RI = rot + 9 * (size_t)r.I;
    const double* RJ = rot + 9 * (size_t)r.J;
    double Rij[9];
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) Rij[3 * a + b] = RJ[3 * a] * RI[3 * b] + RJ[3 * a + 1] * RI[3 * b + 1] + RJ[3 * a + 2] * RI[3 * b + 2];
    K.Rij.insert(K.Rij.end(), Rij, Rij + 9);
    K.u.insert(K.u.end(), u, u + 3);
  }
  return R3D_OK;
}

int translation_averaging(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use, const double* rot,
                          const uint8_t* rot_kept, uint32_t n_views, const r3d_transavg_options& opt, double* centers,
                          double* translations, uint8_t* view_kept, uint8_t* edge_kept, r3d_transavg_summary& S) {
  const double t0 = now_ms();
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::memset(centers, 0, (size_t)n_views * 3 * sizeof(double));
  std::memset(translations, 0, (size_t)n_views * 3 * sizeof(double));
  std::memset(view_kept, 0, n_views);
  if (edge_kept) std::memset(edge_kept, 0, n_rel);
  // ---- 1. the kept edges (select_edges) ----
  const char* fn = "r3d_translation_averaging: ";
  KeptEdges K;
  const int rc0 = select_edges(ctx, fn, rel, n_rel, edge_use, rot, rot_kept, n_views, K);
  S.n_edges = K.n_edges;
  if (rc0) return rc0;
  if (K.kview.empty()) {
    S.ms_host = now_ms() - t0;
    return R3D_OK;
  }
  const std::vector<uint32_t>& kview = K.kview;
  const std::vector<uint2>& kab = K.kab;
  const std::vector<uint2>& ab = K.ab;
  const uint32_t m = (uint32_t)kview.size();
  const bool softl1 = opt.method == kSoftL1;
  std::vector<double> ed;  // per kept edge: chordal u (3, 3 unused); soft-L1 the angle-axis of R_J R_I^T (3), t_IJ / |t_IJ| (3)
  for (size_t k = 0; k < kab.size(); ++k) {
    const double* u = &K.u[3 * k];
    const double* RJ = rot + 9 * (size_t)rel[K.src[k]].J;
    double q[6] = {0, 0, 0, 0, 0, 0};
    if (!softl1) {
      for (int c = 0; c < 3; ++c) q[c] = -(RJ[c] * u[0] + RJ[3 + c] * u[1] + RJ[6 + c] * u[2]);
    } else {
      rp::rotation_to_angle_axis(&K.Rij[9 * k], q);
      for (int c = 0; c < 3; ++c) q[3 + c] = u[c];
    }
    ed.insert(ed.end(), q, q + 6);
    if (edge_kept) edge_kept[K.src[k]] = 1;
  }
  const uint32_t ne = (uint32_t)kab.size();
  S.success = 1;
  S.n_kept_views = m;
  S.n_kept_edges = ne;
  for (uint32_t v : kview) view_kept[v] = 1;
  std::vector<uint32_t> inc_ofs, inc_nbr, inc_edge;
  ra::incidence_lists(m, kab, inc_ofs, inc_nbr, inc_edge);
  // ---- 2. Levenberg-Marquardt ----
  const int N = 3 * ((int)m - 1);            // free view coordinates (view 0 held)
  const uint32_t ns = softl1 ? ne : 0u;      // scales
  const uint32_t Nv = (uint32_t)N + ns;
  const int nblk = (N + kCholNB - 1) / kCholNB;
  std::vector<double> x(Nv);
  for (int j = 0; j < N; ++j) x[j] = softl1 ? 1.0 : start_value((uint64_t)j);
  for (uint32_t e = 0; e < ns; ++e) x[N + e] = 1.0;
  DevArr<uint32_t> d_iofs(w), d_inbr(w), d_iedge(w);
  DevArr<uint2> d_ab(w);
  DevArr<double> d_ed(w), d_A(w), d_L(w), d_Linv(w), d_x(w), d_cur(w), d_trial(w), d_res(w), d_jac(w), d_cost(w), d_scale(w), d_g(w),
      d_diag(w), d_scal(w);
  if (!d_iofs.alloc(m + 1) || !d_inbr.alloc(2 * (size_t)ne) || !d_iedge.alloc(2 * (size_t)ne) || !d_ab.alloc(ne) || !d_ed.alloc(6 * (size_t)ne) ||
      !d_A.alloc((size_t)(N + 1) * N) || !d_L.alloc((size_t)(N + 1) * N + 64) || !d_Linv.alloc((size_t)nblk * kCholNB * kCholNB) ||
      !d_x.alloc(Nv) || !d_cur.alloc(Nv) || !d_trial.alloc(Nv) || !d_res.alloc(3 * (size_t)ne) || !d_jac.alloc(21 * (size_t)ne) ||
      !d_cost.alloc(ne) || !d_scale.alloc(Nv) || !d_g.alloc(Nv) || !d_diag.alloc(Nv) || !d_scal.alloc(8))
    return fail(ctx, R3D_ERR_NOMEM, std::string(fn) + "device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_iofs.p, inc_ofs.data(), (m + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_inbr.p, inc_nbr.data(), inc_nbr.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_iedge.p, inc_edge.data(), inc_edge.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ab.p, ab.data(), ab.size() * sizeof(uint2), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ed.p, ed.data(), ed.size() * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_cur.p, x.data(), Nv * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_scal.p, 0, 8 * sizeof(double), w.stream));
  Events<2> evt;
  R3D_CUDA_TRY(ctx, evt.create());
  R3D_CUDA_TRY(ctx, cudaEventRecord(evt.e[0], w.stream));
  LmParams prm = lm_params(opt.lm);
  if (prm.max_iterations == 0) prm.max_iterations = softl1 ? std::max<uint32_t>(50, 2 * ne) : 500u;
  if (!(prm.function_tolerance > 0.0)) prm.function_tolerance = softl1 ? 1e-6 : 1e-7;
  const double la = opt.softl1_loss;
  const uint32_t eg = (ne + 127) / 128;
  double* cur = d_cur.p;
  double* trial = d_trial.p;
  const ra::AvgBuffers B{d_iofs.p, d_iedge.p, d_ab.p, d_res.p, d_jac.p, d_cost.p, d_scale.p, d_g.p, d_diag.p,
                         d_A.p, d_L.p, d_Linv.p, d_x.p, d_scal.p};
  const int rc = ra::averaging_lm<21>(
      ctx, w, prm, B, ne, 1, Nv, (uint32_t)N, cur, trial, S,
      [&](const double* xx) {
        if (softl1) k_ta_cost<kSoftL1><<<eg, 128, 0, w.stream>>>(xx, d_ab.p, d_ed.p, ne, (uint32_t)N, la, d_cost.p);
        else k_ta_cost<kChordal><<<eg, 128, 0, w.stream>>>(xx, d_ab.p, d_ed.p, ne, (uint32_t)N, la, d_cost.p);
      },
      [&](const double* xx) {
        if (softl1) k_ta_eval<kSoftL1><<<eg, 128, 0, w.stream>>>(xx, d_ab.p, d_ed.p, ne, (uint32_t)N, la, d_res.p, d_jac.p);
        else k_ta_eval<kChordal><<<eg, 128, 0, w.stream>>>(xx, d_ab.p, d_ed.p, ne, (uint32_t)N, la, d_res.p, d_jac.p);
      },
      [&](int mode) {
        if (softl1) k_ta_edge<<<eg, 128, 0, w.stream>>>(mode, d_res.p, d_jac.p, ne, (uint32_t)N, d_scale.p, d_g.p, d_diag.p);
      },
      [&](const double* xx, double inv_radius) {
        k_ta_system<<<m - 1, 128, 0, w.stream>>>(softl1, d_iofs.p, d_inbr.p, d_iedge.p, d_ab.p, d_jac.p, xx, (uint32_t)N, d_scale.p,
                                                 d_g.p, d_diag.p, inv_radius, d_A.p);
      },
      [&](const double* xx, double inv_radius) {
        if (softl1) k_ta_back<<<eg, 128, 0, w.stream>>>(d_ab.p, d_jac.p, xx, d_scale.p, d_g.p, ne, (uint32_t)N, inv_radius, d_x.p);
      });
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaEventRecord(evt.e[1], w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(x.data(), cur, Nv * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  S.ms_solve = evt.ms(0, 1);
  // centres and translations (t = -R C)
  for (uint32_t a = 0; a < m; ++a) {
    const uint32_t v = kview[a];
    const double* R = rot + 9 * (size_t)v;
    double p[3];
    for (int k = 0; k < 3; ++k) p[k] = a == 0 ? 0.0 : x[3 * (size_t)(a - 1) + k];
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
  S.ms_device_total = S.ms_solve;
  S.ms_host = now_ms() - t0 - S.ms_device_total;
  return R3D_OK;
}

}  // namespace ta
}  // namespace r3d

using namespace r3d;

extern "C" void r3d_transavg_default_options(r3d_transavg_options* o) {
  if (!o) return;
  o->method = R3D_TRANSAVG_L2_CHORDAL;
  o->softl1_loss = 0.01;           // SoftLOneLoss(0.01)
  r3d_ba_default_options(&o->lm);
  o->lm.max_iterations = 0;        // the method's cap: 500 (chordal), max(50, 2 x scales) (soft-L1)
  o->lm.function_tolerance = 0.0;  // the method's: 1e-7 (chordal), 1e-6 (soft-L1)
  o->lm.huber_a = 0.0;
  o->lm.refine_intrinsics = 0;
}

extern "C" int r3d_translation_averaging(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                                         const double* rotations, const uint8_t* rot_kept, uint32_t n_views,
                                         const r3d_transavg_options* opt, double* centers, double* translations, uint8_t* view_kept,
                                         uint8_t* edge_kept, r3d_transavg_summary* summary) {
  if (!ctx || (!rel && n_rel) || !opt || (n_views && (!rotations || !rot_kept || !centers || !translations || !view_kept)) || !summary)
    return fail(ctx, R3D_ERR_INVALID, "r3d_translation_averaging: bad arguments");
  std::memset(summary, 0, sizeof(*summary));
  summary->lm_termination = -1;
  if (opt->method == R3D_TRANSAVG_L1)
    return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_translation_averaging: L1 translation averaging is not implemented");
  if (opt->method != R3D_TRANSAVG_L2_CHORDAL && opt->method != R3D_TRANSAVG_SOFTL1)
    return fail(ctx, R3D_ERR_INVALID, "r3d_translation_averaging: unknown method");
  if (opt->method == R3D_TRANSAVG_SOFTL1 && !(opt->softl1_loss > 0.0))
    return fail(ctx, R3D_ERR_INVALID, "r3d_translation_averaging: softl1_loss <= 0");
  return ta::translation_averaging(ctx, rel, n_rel, edge_use, rotations, rot_kept, n_views, *opt, centers, translations, view_kept,
                                   edge_kept, *summary);
}
