// averaging.cuh -- the Levenberg-Marquardt refinement shared by the global-SfM averaging steps, rotations (rotavg.cu) and
// translations (transavg.cu): forward-mode duals, the per-view Jacobi scale and gradient, the step and sum kernels, the
// incidence lists and the host loop around lm_trust_region.cuh's trust region.  Each step keeps its own residuals and
// its own system assembly.  Also the translation steps' shared edge selection (ta::select_edges, transavg.cu) and
// rotavg.cu's 3-column triangular solve (trsm3), which the L1 translation solver (transavg_l1.cu) reuses.  Only for
// translation units compiled with --fmad=false (regard3d_b200/build.py).
#pragma once
#include "r3d_internal.cuh"
#include "lm_trust_region.cuh"

#include <utility>
#include <vector>

namespace r3d {
namespace ra {

// ---- forward-mode duals: value a and N partials ----------------------------------------------------------------
template <int N>
struct Dual {
  static constexpr int kN = N;
  double a;
  double v[N];
};
template <int N> __device__ __forceinline__ Dual<N> dconst(double x) { Dual<N> r; r.a = x; for (int i = 0; i < N; ++i) r.v[i] = 0.0; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator+(const Dual<N>& x, const Dual<N>& y) { Dual<N> r; r.a = x.a + y.a; for (int i = 0; i < N; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator-(const Dual<N>& x, const Dual<N>& y) { Dual<N> r; r.a = x.a - y.a; for (int i = 0; i < N; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator-(const Dual<N>& x) { Dual<N> r; r.a = -x.a; for (int i = 0; i < N; ++i) r.v[i] = -x.v[i]; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator*(const Dual<N>& x, const Dual<N>& y) { Dual<N> r; r.a = x.a * y.a; for (int i = 0; i < N; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator/(const Dual<N>& x, const Dual<N>& y) {
  Dual<N> r; const double inv = 1.0 / y.a; r.a = x.a * inv;
  for (int i = 0; i < N; ++i) r.v[i] = (x.v[i] - r.a * y.v[i]) * inv;
  return r;
}
template <int N> __device__ __forceinline__ Dual<N> operator+(const Dual<N>& x, double s) { Dual<N> r = x; r.a += s; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator-(const Dual<N>& x, double s) { Dual<N> r = x; r.a -= s; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator-(double s, const Dual<N>& x) { Dual<N> r = -x; r.a += s; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator*(const Dual<N>& x, double s) { Dual<N> r; r.a = x.a * s; for (int i = 0; i < N; ++i) r.v[i] = x.v[i] * s; return r; }
template <int N> __device__ __forceinline__ Dual<N> operator*(double s, const Dual<N>& x) { Dual<N> r; r.a = x.a * s; for (int i = 0; i < N; ++i) r.v[i] = x.v[i] * s; return r; }
template <int N> __device__ __forceinline__ Dual<N> sqrt(const Dual<N>& x) { Dual<N> r; r.a = ::sqrt(x.a); const double d = 0.5 / r.a; for (int i = 0; i < N; ++i) r.v[i] = x.v[i] * d; return r; }
template <int N> __device__ __forceinline__ Dual<N> sin(const Dual<N>& x) { Dual<N> r; r.a = ::sin(x.a); const double c = ::cos(x.a); for (int i = 0; i < N; ++i) r.v[i] = c * x.v[i]; return r; }
template <int N> __device__ __forceinline__ Dual<N> cos(const Dual<N>& x) { Dual<N> r; r.a = ::cos(x.a); const double s = -::sin(x.a); for (int i = 0; i < N; ++i) r.v[i] = s * x.v[i]; return r; }
template <int N> __device__ __forceinline__ Dual<N> atan2(const Dual<N>& y, const Dual<N>& x) {
  Dual<N> r; r.a = ::atan2(y.a, x.a); const double d = 1.0 / (x.a * x.a + y.a * y.a);
  for (int i = 0; i < N; ++i) r.v[i] = (x.a * y.v[i] - y.a * x.v[i]) * d;
  return r;
}
// the plain-double forms, so that a residual written once for T = double and T = Dual calls the same names
__device__ __forceinline__ double sqrt(double x) { return ::sqrt(x); }
__device__ __forceinline__ double sin(double x) { return ::sin(x); }
__device__ __forceinline__ double cos(double x) { return ::cos(x); }
__device__ __forceinline__ double atan2(double y, double x) { return ::atan2(y, x); }
template <int N> __device__ __forceinline__ double val(const Dual<N>& x) { return x.a; }
__device__ __forceinline__ double val(double x) { return x; }
template <class T> __device__ __forceinline__ T mk(double x) { return dconst<T::kN>(x); }
template <> __device__ __forceinline__ double mk<double>(double x) { return x; }

// ---- Ceres' angle-axis conversions, for T = double and T = Dual (rotavg.cu, rotavg_l1.cu) ------------------------
// ceres::AngleAxisToRotationMatrix (row-major)
template <class T>
__device__ void aa_to_R(const T* aa, T* R) {
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
// ceres::RotationMatrixToAngleAxis: RotationMatrixToQuaternion + QuaternionToAngleAxis (row-major)
template <class T>
__device__ void R_to_aa(const T* R, T* aa) {
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
// ---- kernels ----------------------------------------------------------------------------------------------------
// All are templates, so that each translation unit that launches one has its own instance.
constexpr int kAvgThreads = 256;  // the one-CTA kernels: k_avg_step, k_avg_sum

// The LM step over Nv variables, one CTA of kThreads (views or rotations first, then from index nb on the scales,
// bounded below by 1; nb = Nv: every variable unbounded): out[0] = 1/2 delta^T (D^2 delta - g) with the unclamped
// delta, out[1] = |x_new - x|^2 with x_new = Plus(x, scaled-back delta) (clamped), out[2] = |x|^2, out[3] =
// max |x - Plus(x, -g / scale)| (the projected unscaled gradient, from the current g).
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_avg_step(const double* __restrict__ delta, const double* __restrict__ g,
                                                       const double* __restrict__ diag, const double* __restrict__ scale,
                                                       const double* __restrict__ x, uint32_t Nv, uint32_t nb, double inv_radius,
                                                       double* __restrict__ x_new, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double mcc = 0.0, dn = 0.0, xn = 0.0, gm = 0.0;
  for (uint32_t j = threadIdx.x; j < Nv; j += kThreads) {
    const double d2 = fmin(fmax(diag[j], 1e-6), 1e32) * inv_radius;
    mcc += delta[j] * (d2 * delta[j] - g[j]);
    const double d = delta[j] * scale[j];
    const double xj = x[j];
    const double gt = g[j] / scale[j];
    if (j < nb) {
      x_new[j] = xj + d;
      dn += d * d;
      gm = fmax(gm, fabs(gt));
    } else {
      const double xc = fmax(xj + d, 1.0);
      x_new[j] = xc;
      dn += (xc - xj) * (xc - xj);
      gm = fmax(gm, fabs(xj - fmax(xj - gt, 1.0)));
    }
    xn += xj * xj;
  }
  mcc = block_sum_fixed<kThreads>(mcc, red);
  dn = block_sum_fixed<kThreads>(dn, red);
  xn = block_sum_fixed<kThreads>(xn, red);
  gm = block_max_fixed<kThreads>(gm, red);
  if (threadIdx.x == 0) {
    out[0] = 0.5 * mcc;
    out[1] = dn;
    out[2] = xn;
    out[3] = gm;
  }
}

// out[0] = sum of v[0..n) (fixed order)
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_avg_sum(const double* __restrict__ v, uint32_t n, double* __restrict__ out) {
  __shared__ double red[kThreads / 32];
  double s = 0.0;
  for (uint32_t i = threadIdx.x; i < n; i += kThreads) s += v[i];
  s = block_sum_fixed<kThreads>(s, red);
  if (threadIdx.x == 0) out[0] = s;
}

// Owner CTA per view a = v0 + blockIdx.x, its incident edges in neighbour order; its variables are 3 blockIdx.x .. +2
// (v0 = 1 when view 0 is held and has none).  An edge's Jacobian is kStride doubles: 3 rows of kStride / 3 columns, the
// edge's first view (ab[e].x) in columns 0..2, its second in 3..5.  mode 0: the Jacobi scale 1 / (1 + ||column||) of
// the view's 3 columns; mode 1: the gradient g = J^T r and diag(J^T J) (scaled).  The walk is latency bound.  With
// no minimum of resident CTAs ptxas fits the kernel into 32 registers and issues each edge's loads only after the
// previous edge is summed, which takes 2.7 times as long; 9 CTAs of 128 threads allow 56 registers, enough to issue
// the loads of several edges together.
template <int kStride>
__global__ void __launch_bounds__(128, 9) k_avg_grad(int mode, const uint32_t* __restrict__ inc_ofs,
                                                     const uint32_t* __restrict__ inc_edge, const uint2* __restrict__ ab,
                                                     const double* __restrict__ res, const double* __restrict__ jac, uint32_t v0,
                                                     double* __restrict__ scale, double* __restrict__ g, double* __restrict__ diag) {
  constexpr int kRow = kStride / 3;
  const uint32_t a = v0 + blockIdx.x, r0 = 3 * blockIdx.x, tid = threadIdx.x;
  const uint32_t b0 = inc_ofs[a], b1 = inc_ofs[a + 1];
  auto col = [&](uint32_t e) -> int { return ab[e].x == a ? 0 : 3; };
  if (mode == 0) {
    if (tid < 3) {
      double n2 = 0.0;
      for (uint32_t p = b0; p < b1; ++p) {
        const uint32_t e = inc_edge[p];
        const int o = col(e) + (int)tid;
        for (int i = 0; i < 3; ++i) n2 += jac[kStride * (size_t)e + kRow * i + o] * jac[kStride * (size_t)e + kRow * i + o];
      }
      scale[r0 + tid] = 1.0 / (1.0 + ::sqrt(n2));
    }
  } else if (tid < 6) {
    const int k = (int)tid % 3;
    const double sk = scale[r0 + k];
    double s = 0.0;
    for (uint32_t p = b0; p < b1; ++p) {
      const uint32_t e = inc_edge[p];
      const int o = col(e) + k;
      for (int i = 0; i < 3; ++i) {
        const double j = jac[kStride * (size_t)e + kRow * i + o] * sk;
        s += tid < 3 ? j * res[3 * (size_t)e + i] : j * j;
      }
    }
    if (tid < 3) g[r0 + k] = s;
    else diag[r0 + k] = s;
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------
// 2-edge-connected components of an undirected multigraph on nodes 0..n-1 (edge k = (eu[k], ev[k]); parallel edges are
// not bridges, self-loops are ignored): bridges by Tarjan's low-link (iterative DFS), then connected components of the
// remaining edges.  Returns the component with the most nodes (>= 2; a tie keeps the one holding the smallest node), or
// -1; comp[v] = component of v, -1 for nodes without edges.
int largest_biedge_component(uint32_t n, const std::vector<uint32_t>& eu, const std::vector<uint32_t>& ev, std::vector<int>& comp);

// rotavg.cu: steps 1 and 2 of both rotation-averaging methods (r3d_rotation_averaging, r3d_rotation_averaging_l1): the
// OK records checked (I != J, ids < n_views, no unordered pair twice) as canonical edges (min, max), triplet rotation
// rejection on the device (k_rotavg_triplets), the largest bi-edge-connected component of the supported edges, local
// ids in view id order (local 0 = the lowest kept view id, the gauge) and the incidence lists.  Zeroes and fills
// view_kept, edge_kept and edge_support (both may be NULL).  R3D_OK with K.kview empty when no component survives;
// R3D_ERR_INVALID for a bad record, R3D_ERR_UNSUPPORTED above kMaxTripletNodes nodes or R3D_ROTAVG_MAX_VIEWS kept views;
// fn prefixes the error messages.
struct KeptComponent {
  uint64_t n_edges = 0, n_triplets = 0, n_valid_triplets = 0;
  double ms_triplets = 0.0;
  std::vector<uint32_t> kview;                      // kept view ids by local id
  std::vector<uint2> kab;                           // kept edges (a < b), in (a, b) order
  std::vector<double> kR;                           // per kept edge R_ab (9, row-major): R_b = R_ab R_a
  std::vector<uint32_t> inc_ofs, inc_nbr, inc_edge;  // incidence_lists of kab
};
int select_component(r3d_ctx* ctx, const char* fn, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                     double max_angular_error_deg, uint8_t* view_kept, uint8_t* edge_kept, uint32_t* edge_support, KeptComponent& K);

// rotavg.cu: L Lt X = Y in place of Y (n x 3 row-major), Z: n x 3 scratch, with the factor L, Linv of dense_cholesky
// (one cooperative launch); trsm3_grid resolves grid 0 and checks that the grid can be co-resident.
int trsm3_grid(r3d_ctx* ctx, DeviceWorker& w, int* grid);
int trsm3(r3d_ctx* ctx, DeviceWorker& w, const double* L, const double* Linv, int n, double* Y, double* Z, int grid);

// Incidence lists of m views over edges given as (lo < hi) and sorted by (lo, hi), in neighbour order: view v's entries
// (lo < v) come first in lo order, then (v, hi > v) in hi order.  ofs: m + 1 offsets; nbr, edge: the neighbour and the
// edge index of each entry.
void incidence_lists(uint32_t m, const std::vector<uint2>& edges, std::vector<uint32_t>& ofs, std::vector<uint32_t>& nbr,
                     std::vector<uint32_t>& edge);

// The device buffers of one refinement, owned by the caller.
struct AvgBuffers {
  const uint32_t* inc_ofs;  // incidence lists (incidence_lists)
  const uint32_t* inc_edge;
  const uint2* ab;          // per edge: the views of Jacobian columns 0..2 and 3..5
  double* res;              // per edge: residual (3) and Jacobian (kStride), written by the eval kernel
  double* jac;
  double* cost;             // per edge: cost term, written by the cost kernel
  double *scale, *g, *diag;  // per variable
  double *A, *L, *Linv;      // the (nb + 1) x nb system (row nb: right-hand side) and its dense_cholesky factor
  double* x;                 // the step (Nv)
  double* scal;              // 8 read-back scalars: k_avg_step's 4, the cost at 4, the not-positive-definite flag at 7
};

// Levenberg-Marquardt from the point in cur over Nv variables: the first nb are the unknowns of the dense system, 3 per
// view from view v0 on; from nb on, scales bounded below by 1 that the caller's after-solve hook steps.  ne: edges.
// The hooks only launch kernels on w.stream:
//   cost(x)                  the cost terms at x into B.cost
//   eval(x)                  residuals and Jacobians at x into B.res / B.jac
//   cols(mode)               after each k_avg_grad: the same mode for variables nb.. (scale, or gradient and diag)
//   assemble(x, inv_radius)  the scaled system J^T J + D^2 / radius | -g into the zeroed B.A
//   solved(x, inv_radius)    after the solve of B.x[0..nb): the steps of variables nb..
// On return cur holds the solution and S its lm_* fields.
template <int kStride, class Summary, class Cost, class Eval, class Cols, class Assemble, class Solved>
int averaging_lm(r3d_ctx* ctx, DeviceWorker& w, const LmParams& prm, const AvgBuffers& B, uint32_t ne, uint32_t v0, uint32_t Nv,
                 uint32_t nb, double*& cur, double*& trial, Summary& S, Cost cost, Eval eval, Cols cols, Assemble assemble,
                 Solved solved) {
  const int N = (int)nb;
  double scal[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  auto read_scal = [&]() -> int {
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(scal, B.scal, sizeof(scal), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    return R3D_OK;
  };
  auto eval_cost = [&](const double* x, double* out) -> int {
    cost(x);
    k_avg_sum<kAvgThreads><<<1, kAvgThreads, 0, w.stream>>>(B.cost, ne, B.scal + 4);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    int rc;
    if ((rc = read_scal())) return rc;
    *out = scal[4];
    return R3D_OK;
  };
  bool have_scale = false;
  double gmax = 0.0;
  auto evaluate = [&]() -> int {  // residuals, Jacobians, the scale on the first call, g, diag and the projected gradient
    eval(cur);
    if (!have_scale) {
      k_avg_grad<kStride><<<nb / 3, 128, 0, w.stream>>>(0, B.inc_ofs, B.inc_edge, B.ab, B.res, B.jac, v0, B.scale, B.g, B.diag);
      cols(0);
      have_scale = true;
    }
    k_avg_grad<kStride><<<nb / 3, 128, 0, w.stream>>>(1, B.inc_ofs, B.inc_edge, B.ab, B.res, B.jac, v0, B.scale, B.g, B.diag);
    cols(1);
    // the step kernel with a zero step and radius reports the projected gradient in scal[3]
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(B.x, 0, Nv * sizeof(double), w.stream));
    k_avg_step<kAvgThreads><<<1, kAvgThreads, 0, w.stream>>>(B.x, B.g, B.diag, B.scale, cur, Nv, nb, 0.0, trial, B.scal);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    int rc;
    if ((rc = read_scal())) return rc;
    gmax = scal[3];
    return R3D_OK;
  };
  int rc;
  double f = 0.0;
  if ((rc = eval_cost(cur, &f))) return rc;
  S.lm_initial_cost = f;
  LmTrustRegion lm(prm);
  if ((rc = evaluate())) return rc;
  const bool stop = lm.start(gmax);
  for (uint32_t iter = 1; !stop && iter <= lm.p.max_iterations; ++iter) {
    lm.iterations = iter;
    const double inv_radius = 1.0 / lm.radius;
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(B.A, 0, (size_t)(N + 1) * N * sizeof(double), w.stream));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(B.scal + 7, 0, sizeof(double), w.stream));
    assemble(cur, inv_radius);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if ((rc = dense_cholesky(ctx, w, B.A, B.L, B.Linv, N, B.scal + 7, B.x))) return rc;
    solved(cur, inv_radius);
    k_avg_step<kAvgThreads><<<1, kAvgThreads, 0, w.stream>>>(B.x, B.g, B.diag, B.scale, cur, Nv, nb, inv_radius, trial, B.scal);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if ((rc = read_scal())) return rc;
    const double model_cost_change = scal[0];
    bool accepted = false;
    if (lm.step_usable(scal[7] == 0.0, model_cost_change)) {
      if (lm.step_too_small(scal[1], scal[2])) break;
      double new_f = 0.0;
      if ((rc = eval_cost(trial, &new_f))) return rc;
      if ((accepted = lm.accept(f, new_f, model_cost_change))) {
        std::swap(cur, trial);
        f = new_f;
        if ((rc = evaluate())) return rc;
        if (lm.converged(gmax)) break;
      }
    }
    if (!accepted && lm.reject()) break;
  }
  S.lm_iterations = lm.iterations;
  S.lm_successful_steps = lm.successful;
  S.lm_termination = lm.termination;
  S.lm_final_cost = f;
  return R3D_OK;
}

}  // namespace ra

namespace ta {

// The edges of a translation-averaging call (transavg.cu), shared by r3d_translation_averaging and
// r3d_translation_averaging_l1: the OK records with edge_use set, checked (I != J, ids < n_views, a non-zero finite
// translation, no unordered pair twice), in canonical (min, max) order, both views rotation-kept; the largest
// bi-edge-connected component of them, local ids in view id order (local 0 = the lowest kept view id, the gauge).
struct KeptEdges {
  uint64_t n_edges = 0;          // usable edges before the component
  std::vector<uint32_t> kview;   // kept view ids by local id; empty: no component
  std::vector<uint2> kab, ab;    // per kept edge: canonical (lo < hi) and record-oriented (I, J) local ids
  std::vector<uint64_t> src;     // per kept edge: its record
  std::vector<double> Rij, u;    // per kept edge: R_J R_I^T (9, row-major) and t_IJ / |t_IJ| (3)
};
// R3D_OK (K.kview empty when no component survives), R3D_ERR_INVALID for a bad record, R3D_ERR_UNSUPPORTED for more
// than R3D_ROTAVG_MAX_VIEWS kept views; fn prefixes the error messages.
int select_edges(r3d_ctx* ctx, const char* fn, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                 const double* rot, const uint8_t* rot_kept, uint32_t n_views, KeptEdges& K);

}  // namespace ta
}  // namespace r3d
