// resection.cu -- absolute pose of views from 2D-3D correspondences (r3d_resect_views, r3d_sfm_resect_views).
// COMPILED WITH --fmad=false (regard3d_b200/build.py): the undistorted pixels, the P3P models and every AC-RANSAC
// decision must equal the CPU restatement's (oracle/oracle_resection.cpp) bit for bit; the pose refinement follows its
// LM decisions.
//
// Replaces SfM_Localizer::Localize + SfM_Localizer::RefinePose (OpenMVG 1.4 sfm_localizer.cpp), the first step of the
// loop both incremental engines run (src/threads/R3DTriangulationThread.cpp:416-512).  Three stages per device, one
// stream, one synchronisation:
//   1. k_resect_points, one thread per correspondence: the pixel undistorted once by the inverse of the view's camera
//      model (p3p.cuh), the structure point split into the layout the AC-RANSAC kernel reads;
//   2. k_acransac_fused<3>: the filters' persistent one-CTA-per-problem AC-RANSAC with the P3P solver and the pinhole
//      reprojection error (acransac_fused.cu), one launch per size class; it hands back P = K [R | t] of the best model;
//   3. k_resect_refine, one persistent CTA per view: Levenberg-Marquardt on the six pose parameters over the AC-RANSAC
//      inliers, residuals on the original pixels through the full camera model (ba_model.cuh), Huber loss, the trust
//      region of the bundle adjustment.  The 6 x 6 normal equations are reduced in a fixed order (no floating-point
//      atomics), so a call is reproducible.  FP64 throughout; bound by FP64 latency, not by tensor cores or HBM.
#include "acransac.cuh"
#include "ba_model.cuh"
#include "detmath.cuh"
#include "lm_trust_region.cuh"
#include "p3p.cuh"
#include "relpose_math.cuh"
#include "r3d_sfm.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

namespace r3d {

namespace {

struct RsView {            // a view that reached the AC-RANSAC stage (device)
  uint32_t ofs, M;         // its correspondences in the device arrays
  int model;               // R3D_CAM_*
  int pad_;
  double intr[6], ext[2];  // f, ppx, ppy, the model's first three distortion coefficients | coefficients 4, 5
};

struct RsLm {              // refinement result
  double pose[6];          // angle-axis | t
  uint32_t iterations, successful;
  int termination;         // -1: not refined
  int pad_;
  double initial_cost, final_cost;
};

// [R | t] of P = K [R | t], K = [f 0 ppx; 0 f ppy; 0 0 1]
__host__ __device__ inline void pose_from_projective(const double* K, const double* P, double* R, double* t) {
  for (int j = 0; j < 3; ++j) {
    R[6 + j] = P[8 + j];
    R[j] = (P[j] - K[1] * P[8 + j]) / K[0];
    R[3 + j] = (P[4 + j] - K[2] * P[8 + j]) / K[0];
  }
  t[2] = P[11];
  t[0] = (P[3] - K[1] * P[11]) / K[0];
  t[1] = (P[7] - K[2] * P[11]) / K[0];
}

// ---- 1. undistortion and the AC-RANSAC point layout ------------------------------------------------------------------
// grid (8, views): X (3 per correspondence) -> x1 = (X, Y), x3 = Z; x (2 per correspondence) -> x2 = undistorted pixel;
// idm = (i, i): the kernel lists a problem's inliers by copying entries of this array
__global__ void __launch_bounds__(256) k_resect_points(const RsView* __restrict__ views, const double* __restrict__ X,
                                                       const double2* __restrict__ x, double2* __restrict__ x1,
                                                       double* __restrict__ x3, double2* __restrict__ x2, uint2* __restrict__ idm) {
  const RsView& v = views[blockIdx.y];
  const double disto[5] = {v.intr[3], v.intr[4], v.intr[5], v.ext[0], v.ext[1]};
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < v.M; i += gridDim.x * blockDim.x) {
    const size_t g = (size_t)v.ofs + i;
    x1[g] = make_double2(X[3 * g], X[3 * g + 1]);
    x3[g] = X[3 * g + 2];
    const double2 o = x[g];
    double ux, uy;
    p3p::undistort_pixel(v.model, v.intr[0], v.intr[1], v.intr[2], disto, o.x, o.y, &ux, &uy);
    x2[g] = make_double2(ux, uy);
    idm[g] = make_uint2(i, i);
  }
}

// ---- 3. pose-only Levenberg-Marquardt ------------------------------------------------------------------------------------
constexpr int kRThreads = 256;
constexpr int kRWarps = kRThreads / 32;
constexpr int kREntries = 27;            // 21 lower-triangle entries of J^T J + 6 of J^T r

struct RefineSmem {
  double pose[6], pose_new[6], scale[6], g[6], diag[6], D2[6], delta[6];
  double H[36];
  double part[kRWarps][kREntries + 1];
  double sums[kREntries + 1];
  RsView view;
  int pd;
  uint32_t work;
};

// sums[e] = sum over the threads of v[e], e < n: a fixed shuffle tree per warp, then the warps in order
__device__ void block_sums(const double* v, int n, RefineSmem& S) {
  for (int e = 0; e < n; ++e) {
    double a = v[e];
    for (int o = 16; o >= 1; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if ((threadIdx.x & 31u) == 0) S.part[threadIdx.x >> 5][e] = a;
  }
  __syncthreads();
  if ((int)threadIdx.x < n) {
    double s = 0.0;
    for (int w = 0; w < kRWarps; ++w) s += S.part[w][threadIdx.x];
    S.sums[threadIdx.x] = s;
  }
  __syncthreads();
}

// one persistent CTA per view; order: view slots, most correspondences first.  The inliers of slot a are
// inl[views[a].ofs + 0 .. fo[a].n_inliers) (indices into the view's correspondences, AC-RANSAC's residual order).
__global__ void __launch_bounds__(kRThreads) k_resect_refine(const RsView* __restrict__ views, const uint32_t* __restrict__ order,
                                                             uint32_t n_order, uint32_t* __restrict__ work_counter,
                                                             const AcFusedOut* __restrict__ fo, const double* __restrict__ models,
                                                             const uint2* __restrict__ inl, const double2* __restrict__ x1,
                                                             const double* __restrict__ x3, const double2* __restrict__ xo,
                                                             RsLm* __restrict__ out, LmParams prm) {
  __shared__ RefineSmem S;
  const uint32_t tid = threadIdx.x;
  for (;;) {
    __syncthreads();
    if (tid == 0) S.work = atomicAdd(work_counter, 1u);
    __syncthreads();
    const uint32_t wk = S.work;
    if (wk >= n_order) break;
    const uint32_t a = order[wk];
    const AcFusedOut f = fo[a];
    if (!(f.minNFA < 0.0) || !((double)f.n_inliers > 2.5 * 3)) continue;  // no model: nothing to refine
    if (tid == 0) {
      S.view = views[a];
      double R[9], t[3];
      pose_from_projective(S.view.intr, models + 12 * (size_t)a, R, t);
      rp::rotation_to_angle_axis(R, S.pose);
      for (int i = 0; i < 3; ++i) S.pose[3 + i] = t[i];
    }
    __syncthreads();
    const uint32_t N = f.n_inliers;
    const size_t base = S.view.ofs;
    const int model = S.view.model;

    auto total_cost = [&](const double* pose) -> double {
      double c = 0.0;
      for (uint32_t p = tid; p < N; p += kRThreads) {
        const size_t g = base + inl[base + p].x;
        const double2 xy = x1[g], ob = xo[g];
        const double X[3] = {xy.x, xy.y, x3[g]};
        double r[2], rho1;
        ba::residual_only(model, S.view.intr, S.view.ext, pose, X, ob.x, ob.y, r);
        c += 0.5 * ba::huber_rho(r[0] * r[0] + r[1] * r[1], prm.huber_a, &rho1);
      }
      block_sums(&c, 1, S);
      return S.sums[0];
    };
    // Corrector-scaled residuals and pose Jacobians at S.pose: the Jacobi scale on the first call, then g = J^T r and
    // H = J^T J of the scaled columns
    auto evaluate = [&](bool first) {
      if (first) {
        double n2[6] = {0, 0, 0, 0, 0, 0};
        for (uint32_t p = tid; p < N; p += kRThreads) {
          const size_t g = base + inl[base + p].x;
          const double2 xy = x1[g], ob = xo[g];
          const double X[3] = {xy.x, xy.y, x3[g]};
          double r[2], Ji[12], Jc[12], Jp[6], rho1;
          ba::residual_jacobian(model, S.view.intr, S.view.ext, S.pose, X, ob.x, ob.y, r, Ji, Jc, Jp);
          ba::huber_rho(r[0] * r[0] + r[1] * r[1], prm.huber_a, &rho1);
          const double sq = sqrt(rho1);
          for (int k = 0; k < 6; ++k) {
            const double j0 = Jc[k] * sq, j1 = Jc[6 + k] * sq;
            n2[k] += j0 * j0 + j1 * j1;
          }
        }
        block_sums(n2, 6, S);
        if (tid < 6) S.scale[tid] = 1.0 / (1.0 + sqrt(S.sums[tid]));
        __syncthreads();
      }
      double acc[kREntries];
      for (int e = 0; e < kREntries; ++e) acc[e] = 0.0;
      for (uint32_t p = tid; p < N; p += kRThreads) {
        const size_t g = base + inl[base + p].x;
        const double2 xy = x1[g], ob = xo[g];
        const double X[3] = {xy.x, xy.y, x3[g]};
        double r[2], Ji[12], Jc[12], Jp[6], rho1;
        ba::residual_jacobian(model, S.view.intr, S.view.ext, S.pose, X, ob.x, ob.y, r, Ji, Jc, Jp);
        ba::huber_rho(r[0] * r[0] + r[1] * r[1], prm.huber_a, &rho1);
        const double sq = sqrt(rho1);
        const double r0 = r[0] * sq, r1 = r[1] * sq;
        double j0[6], j1[6];
        for (int k = 0; k < 6; ++k) {
          j0[k] = Jc[k] * sq * S.scale[k];
          j1[k] = Jc[6 + k] * sq * S.scale[k];
        }
        int e = 0;
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j <= i; ++j) acc[e++] += j0[i] * j0[j] + j1[i] * j1[j];
        for (int k = 0; k < 6; ++k) acc[21 + k] += j0[k] * r0 + j1[k] * r1;
      }
      block_sums(acc, kREntries, S);
      if (tid == 0) {
        int e = 0;
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j <= i; ++j) S.H[6 * i + j] = S.sums[e++];
        for (int k = 0; k < 6; ++k) { S.g[k] = S.sums[21 + k]; S.diag[k] = S.H[7 * k]; }
      }
      __syncthreads();
    };
    auto grad_max = [&]() -> double {
      double m = 0.0;
      for (int j = 0; j < 6; ++j) m = fmax(m, fabs(S.g[j] / S.scale[j]));
      return m;
    };

    double cost = total_cost(S.pose);
    const double initial_cost = cost;
    LmTrustRegion lm(prm);  // every thread keeps its own: the inputs are block-wide, so are the decisions
    evaluate(true);
    if (!lm.start(grad_max()))
      for (uint32_t iter = 1; iter <= prm.max_iterations; ++iter) {
        lm.iterations = iter;
        __syncthreads();
        if (tid == 0) {  // LevenbergMarquardtStrategy: (H + D^2) delta = -g, D^2 = clamp(diag, 1e-6, 1e32) / radius
          double A[36], b[6];
          for (int j = 0; j < 6; ++j) S.D2[j] = fmin(fmax(S.diag[j], 1e-6), 1e32) / lm.radius;
          for (int i = 0; i < 6; ++i) {
            for (int j = 0; j <= i; ++j) A[6 * i + j] = S.H[6 * i + j] + (i == j ? S.D2[i] : 0.0);
            b[i] = -S.g[i];
          }
          S.pd = chol_solve_small<6>(A, b);
          if (S.pd)
            for (int j = 0; j < 6; ++j) S.delta[j] = b[j];
        }
        __syncthreads();
        const bool pd = S.pd != 0;
        double model_cost_change = 0.0;
        if (pd) {
          double m = 0.0;
          for (int j = 0; j < 6; ++j) m += S.delta[j] * (S.D2[j] * S.delta[j] - S.g[j]);
          model_cost_change = 0.5 * m;
        }
        bool accepted = false;
        if (lm.step_usable(pd, model_cost_change)) {
          double dn = 0.0, xn = 0.0;
          for (int j = 0; j < 6; ++j) {
            const double d = S.delta[j] * S.scale[j];
            dn += d * d;
            xn += S.pose[j] * S.pose[j];
          }
          if (tid < 6) S.pose_new[tid] = S.pose[tid] + S.delta[tid] * S.scale[tid];
          __syncthreads();
          if (lm.step_too_small(dn, xn)) break;
          const double new_cost = total_cost(S.pose_new);
          if ((accepted = lm.accept(cost, new_cost, model_cost_change))) {
            if (tid < 6) S.pose[tid] = S.pose_new[tid];
            cost = new_cost;
            __syncthreads();
            evaluate(false);
            if (lm.converged(grad_max())) break;
          }
        }
        if (!accepted && lm.reject()) break;
      }
    __syncthreads();
    if (tid == 0) {
      RsLm o;
      for (int k = 0; k < 6; ++k) o.pose[k] = S.pose[k];
      o.iterations = lm.iterations;
      o.successful = lm.successful;
      o.termination = lm.termination;
      o.pad_ = 0;
      o.initial_cost = initial_cost;
      o.final_cost = cost;
      out[a] = o;
    }
  }
}

void set_pose(r3d_resection& o, const double* R, const double* t) {
  std::memcpy(o.rotation, R, sizeof(o.rotation));
  std::memcpy(o.translation, t, sizeof(o.translation));
  r3d_sfm::center_of(R, t, o.center);
}

// views [v0, v1) on worker w; inl[v]: the view's AC-RANSAC inliers (residual order)
int resect_range(r3d_ctx* ctx, DeviceWorker& w, const r3d_resection_view* views, uint32_t v0, uint32_t v1, const double* X,
                 const double* x, const r3d_resection_options& opt, r3d_resection* out, std::vector<std::vector<uint32_t>>& inl,
                 r3d_resection_timing& T) {
  const double t0 = now_ms();
  T = r3d_resection_timing{};
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::vector<uint32_t> cand;
  for (uint32_t v = v0; v < v1; ++v) {
    r3d_resection& o = out[v];
    std::memset(&o, 0, sizeof(o));
    o.view_id = views[v].view_id;
    o.lm_termination = -1;
    o.status = views[v].count <= 3 ? R3D_RESECT_TOO_FEW
               : !(views[v].intrinsic.focal > 0.0) ? R3D_RESECT_NO_INTRINSIC
                                                    : R3D_RESECT_NO_MODEL;
    if (o.status == R3D_RESECT_NO_MODEL) cand.push_back(v);
  }
  if (cand.empty()) {
    T.ms_host = now_ms() - t0;
    return R3D_OK;
  }
  const uint32_t n = (uint32_t)cand.size();
  // ---- per view set-up: the a-contrario adaptor for resection with known K (point-to-point, pixel units) ----
  std::vector<AcPair> hpairs(n);
  std::vector<RsView> hviews(n);
  uint64_t pt_total = 0, tbl_total = 0;
  uint32_t maxM = 0;
  for (uint32_t a = 0; a < n; ++a) {
    const r3d_resection_view& v = views[cand[a]];
    const uint32_t M = (uint32_t)v.count;
    AcPair& ap = hpairs[a];
    std::memset(&ap, 0, sizeof(ap));
    ap.pt_ofs = (uint32_t)pt_total; ap.M = M; ap.tbl_ofs = (uint32_t)tbl_total;
    ap.max_thr = opt.precision_px * opt.precision_px;  // upper_bound_precision = Square(error_max)
    ap.logalpha0 = dm::log10_det(R3D_PI / ((double)v.width * (double)v.height));
    ap.loge0 = dm::log10_det((double)ac_max_models(3) * (double)(M - ac_min_samples(3)));
    ap.K[0] = v.intrinsic.focal; ap.K[1] = v.intrinsic.ppx; ap.K[2] = v.intrinsic.ppy;
    ap.K[3] = (double)v.width * (double)v.width + (double)v.height * (double)v.height;
    RsView& rv = hviews[a];
    std::memset(&rv, 0, sizeof(rv));
    rv.ofs = ap.pt_ofs; rv.M = M; rv.model = v.intrinsic.model;
    rv.intr[0] = v.intrinsic.focal; rv.intr[1] = v.intrinsic.ppx; rv.intr[2] = v.intrinsic.ppy;
    for (int i = 0; i < 3; ++i) rv.intr[3 + i] = v.intrinsic.disto[i];
    rv.ext[0] = v.intrinsic.disto[3]; rv.ext[1] = v.intrinsic.disto[4];
    pt_total += M;
    tbl_total += M + 2;
    maxM = std::max(maxM, M);
  }
  if (pt_total > 0xfffffff0ull) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: too many correspondences in one call");
  std::vector<double> hX(3 * pt_total), hx(2 * pt_total);
  parallel_for(ctx->host_threads, n, [&](size_t a) {
    const r3d_resection_view& v = views[cand[a]];
    std::memcpy(&hX[3 * (size_t)hpairs[a].pt_ofs], X + 3 * v.first, 3 * v.count * sizeof(double));
    std::memcpy(&hx[2 * (size_t)hpairs[a].pt_ofs], x + 2 * v.first, 2 * v.count * sizeof(double));
  });
  // ---- the persistent AC-RANSAC kernel's tables, size classes and scratch ----
  AcTables tab(w);
  AcFused fused(w);
  int rc = tab.upload(ctx, w, ac_min_samples(3), maxM, tbl_total);
  if (rc) return rc;
  rc = fused.plan(ctx, w, 3, hpairs);
  if (rc) return rc;
  std::vector<uint32_t> lm_order(n);  // refinement: most correspondences first
  for (uint32_t a = 0; a < n; ++a) lm_order[a] = a;
  std::stable_sort(lm_order.begin(), lm_order.end(), [&](uint32_t p, uint32_t q) { return hpairs[p].M > hpairs[q].M; });

  DevArr<AcPair> d_pairs(w);
  DevArr<RsView> d_views(w);
  DevArr<double> d_X(w), d_x3(w), d_model(w);
  DevArr<double2> d_xo(w), d_x1(w), d_x2(w);
  DevArr<uint2> d_idm(w), d_outm(w);
  DevArr<uint32_t> d_lm_order(w), d_lm_work(w);
  DevArr<AcFusedOut> d_out(w);
  DevArr<RsLm> d_lm(w);
  if (!d_pairs.alloc(n) || !d_views.alloc(n) || !d_X.alloc(3 * pt_total) || !d_x3.alloc(pt_total) || !d_xo.alloc(pt_total) ||
      !d_x1.alloc(pt_total) || !d_x2.alloc(pt_total) || !d_idm.alloc(pt_total) || !d_outm.alloc(pt_total) ||
      !d_lm_order.alloc(n) || !d_lm_work.alloc(1) || !d_model.alloc(12 * (size_t)n) || !d_out.alloc(n) || !d_lm.alloc(n))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_resect_views: device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_pairs.p, hpairs.data(), n * sizeof(AcPair), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_views.p, hviews.data(), n * sizeof(RsView), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_X.p, hX.data(), hX.size() * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_xo.p, hx.data(), hx.size() * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_lm_order.p, lm_order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_lm_work.p, 0, sizeof(uint32_t), w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_lm.p, 0xff, n * sizeof(RsLm), w.stream));  // termination -1: not refined
  Events<3> ev;
  R3D_CUDA_TRY(ctx, ev.create());
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[0], w.stream));
  for (uint32_t a0 = 0; a0 < n; a0 += 65535u) {  // gridDim.y limit
    const uint32_t na = std::min(65535u, n - a0);
    k_resect_points<<<dim3(8, na), 256, 0, w.stream>>>(d_views.p + a0, d_X.p, d_xo.p, d_x1.p, d_x3.p, d_x2.p, d_idm.p);
    T.kernel_launches += 1;
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  rc = launch_ac_tables(ctx, w, d_pairs.p, n, tab.vlog10.p, tab.logc_n.p);
  if (rc) return rc;
  T.kernel_launches += 1;
  rc = fused.launch(ctx, w, d_pairs.p, d_x1.p, d_x2.p, d_x3.p, tab.logc_n.p, tab.logc_k.p, opt.max_iter, d_idm.p, d_outm.p, d_out.p,
                    d_model.p, T.kernel_launches);
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[1], w.stream));
  if (opt.refine) {
    const uint32_t grid = std::min<uint32_t>(n, (uint32_t)w.sm_count);
    k_resect_refine<<<grid, kRThreads, 0, w.stream>>>(d_views.p, d_lm_order.p, n, d_lm_work.p, d_out.p, d_model.p, d_outm.p,
                                                      d_x1.p, d_x3.p, d_xo.p, d_lm.p, lm_params(opt.ba));
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    T.kernel_launches += 1;
  }
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[2], w.stream));
  std::vector<AcFusedOut> hout(n);
  std::vector<double> hmodel(12 * (size_t)n);
  std::vector<RsLm> hlm(n);
  std::vector<uint2> houtm(pt_total);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hout.data(), d_out.p, n * sizeof(AcFusedOut), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hmodel.data(), d_model.p, hmodel.size() * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hlm.data(), d_lm.p, n * sizeof(RsLm), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(houtm.data(), d_outm.p, pt_total * sizeof(uint2), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  T.ms_ransac = ev.ms(0, 1);
  T.ms_refine = ev.ms(1, 2);
  T.ms_device_total = T.ms_ransac + T.ms_refine;
  for (uint32_t a = 0; a < n; ++a) {
    const AcFusedOut& f = hout[a];
    if (!(f.minNFA < 0.0) || !((double)f.n_inliers > 2.5 * 3)) continue;  // R3D_RESECT_NO_MODEL stays
    r3d_resection& o = out[cand[a]];
    o.status = R3D_RESECT_OK;
    o.n_inliers = f.n_inliers;
    o.found_residual_precision = std::sqrt(f.errorMax);
    pose_from_projective(hpairs[a].K, &hmodel[12 * (size_t)a], o.rotation_ransac, o.translation_ransac);
    set_pose(o, o.rotation_ransac, o.translation_ransac);
    std::vector<uint32_t>& il = inl[cand[a]];
    il.resize(f.n_inliers);
    for (uint32_t k = 0; k < f.n_inliers; ++k) il[k] = houtm[(size_t)hpairs[a].pt_ofs + k].x;
    if (!opt.refine) continue;
    const RsLm& l = hlm[a];
    o.lm_iterations = l.iterations;
    o.lm_successful_steps = l.successful;
    o.lm_termination = l.termination;
    o.lm_initial_cost = l.initial_cost;
    o.lm_final_cost = l.final_cost;
    T.lm_iterations += l.iterations;
    if (l.termination == 4) continue;  // the solve failed: the AC-RANSAC pose stays
    double R[9];
    r3d_sfm::angle_axis_to_rotation(l.pose, R);
    set_pose(o, R, l.pose + 3);
  }
  T.ms_host = now_ms() - t0 - T.ms_device_total;
  return R3D_OK;
}

bool finite_all(const double* p, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

}  // namespace

}  // namespace r3d

using namespace r3d;

extern "C" void r3d_resection_default_options(r3d_resection_options* o) {
  if (!o) return;
  o->precision_px = std::numeric_limits<double>::infinity();  // SfM_Localizer: error_max = infinity, pure a-contrario
  o->max_iter = 4096;
  o->refine = 1;
  r3d_ba_default_options(&o->ba);
  o->ba.refine_intrinsics = 0;  // RefinePose(b_refine_pose = true, b_refine_intrinsic = false)
}

extern "C" int r3d_resect_views(r3d_ctx* ctx, const r3d_resection_view* views, uint32_t n_views, const double* X, const double* x,
                                const r3d_resection_options* opt, r3d_resection* out, uint32_t* inliers, uint64_t* inlier_ofs) {
  if (!ctx || !opt || (n_views && (!views || !out))) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: bad arguments");
  if (inliers && !inlier_ofs) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: inliers without inlier_ofs");
  if (!(opt->precision_px > 0.0) || opt->max_iter == 0) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: bad AC-RANSAC options");
  if (opt->refine && opt->ba.refine_intrinsics)
    return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: the pose refinement keeps the intrinsics fixed");
  for (uint32_t v = 0; v < n_views; ++v) {
    const r3d_resection_view& rv = views[v];
    if (rv.count > 0xfffffff0ull) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: too many correspondences in one view");
    if (rv.count && (!X || !x)) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: bad arguments");
    if (rv.width == 0 || rv.height == 0) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: a view without a size");
    if (rv.intrinsic.focal > 0.0) {
      const int m = rv.intrinsic.model;
      if (m < R3D_CAM_PINHOLE || m > R3D_CAM_PINHOLE_FISHEYE) return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: unknown camera model");
      if (!std::isfinite(rv.intrinsic.focal) || !std::isfinite(rv.intrinsic.ppx) || !std::isfinite(rv.intrinsic.ppy) ||
          !finite_all(rv.intrinsic.disto, 5))
        return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: non-finite intrinsic");
    }
    if (!finite_all(X + 3 * rv.first, 3 * rv.count) || !finite_all(x + 2 * rv.first, 2 * rv.count))
      return fail(ctx, R3D_ERR_INVALID, "r3d_resect_views: non-finite correspondence");
  }
  std::vector<std::vector<uint32_t>> inl(n_views);
  // the views are independent: contiguous ranges of equal correspondence counts, one per device (the rule of
  // r3d_relative_poses)
  const std::vector<uint64_t> cut = balanced_cuts(n_views, ctx->workers.size(), [&](uint64_t v) { return views[v].count; });
  std::vector<r3d_resection_timing> tms(ctx->workers.size());
  const int rc = fan_out(ctx, [&](size_t k, DeviceWorker& w) {
    return resect_range(ctx, w, views, (uint32_t)cut[k], (uint32_t)cut[k + 1], X, x, *opt, out, inl, tms[k]);
  });
  if (rc) return rc;
  r3d_resection_timing sum{};
  for (const r3d_resection_timing& t : tms) {
    sum.ms_ransac = std::max(sum.ms_ransac, t.ms_ransac);
    sum.ms_refine = std::max(sum.ms_refine, t.ms_refine);
    sum.ms_device_total = std::max(sum.ms_device_total, t.ms_device_total);
    sum.ms_host = std::max(sum.ms_host, t.ms_host);
    sum.kernel_launches += t.kernel_launches;
    sum.lm_iterations += t.lm_iterations;
  }
  ctx->resection_timing = sum;
  if (inlier_ofs) {
    uint64_t ofs = 0;
    for (uint32_t v = 0; v < n_views; ++v) {
      inlier_ofs[v] = ofs;
      if (inliers) std::memcpy(inliers + ofs, inl[v].data(), inl[v].size() * sizeof(uint32_t));
      ofs += inl[v].size();
    }
    inlier_ofs[n_views] = ofs;
  }
  return R3D_OK;
}

extern "C" int r3d_sfm_resect_views(r3d_ctx* ctx, r3d_sfm_data* sd, const uint32_t* view_ids, uint32_t n,
                                    const r3d_resection_options* opt, r3d_resection* out, uint32_t* n_out) {
  if (!ctx || !sd || !opt || (n && !view_ids)) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_resect_views: bad arguments");
  if (n_out) *n_out = 0;
  std::vector<uint32_t> ids;
  if (n) {
    ids.assign(view_ids, view_ids + n);
  } else {
    for (const auto& kv : sd->views)
      if (!sd->poses.count(kv.second.id_pose)) ids.push_back(kv.first);
  }
  if (ids.size() && !out) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_resect_views: bad arguments");
  std::vector<r3d_resection_view> rv(ids.size());
  std::map<uint32_t, uint32_t> slot;  // view id -> index in rv
  for (size_t k = 0; k < ids.size(); ++k) {
    const auto vit = sd->views.find(ids[k]);
    if (vit == sd->views.end()) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_resect_views: unknown view id");
    if (sd->poses.count(vit->second.id_pose)) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_resect_views: the view already has a pose");
    if (!slot.emplace(ids[k], (uint32_t)k).second) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_resect_views: a view id given twice");
    const auto iit = sd->intrinsics.find(vit->second.id_intrinsic);
    if (iit == sd->intrinsics.end()) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_resect_views: unknown intrinsic id");
    r3d_resection_view& r = rv[k];
    std::memset(&r, 0, sizeof(r));
    r.view_id = ids[k];
    r.width = vit->second.width;
    r.height = vit->second.height;
    r3d_sfm::to_c_intrinsic(iit->first, iit->second, &r.intrinsic);
  }
  // the 2D-3D correspondences of a view: every landmark that holds an observation of it, in landmark-id order
  std::vector<std::vector<double>> Xs(ids.size()), xs(ids.size());
  for (const auto& lm : sd->structure)
    for (const auto& ob : lm.second.obs) {
      const auto s = slot.find(ob.first);
      if (s == slot.end()) continue;
      Xs[s->second].insert(Xs[s->second].end(), lm.second.X, lm.second.X + 3);
      xs[s->second].insert(xs[s->second].end(), ob.second.x, ob.second.x + 2);
    }
  std::vector<double> X, x;
  for (size_t k = 0; k < ids.size(); ++k) {
    rv[k].first = x.size() / 2;
    rv[k].count = xs[k].size() / 2;
    X.insert(X.end(), Xs[k].begin(), Xs[k].end());
    x.insert(x.end(), xs[k].begin(), xs[k].end());
  }
  X.resize(std::max<size_t>(X.size(), 3));
  x.resize(std::max<size_t>(x.size(), 2));
  const int rc = r3d_resect_views(ctx, rv.data(), (uint32_t)rv.size(), X.data(), x.data(), opt, out, nullptr, nullptr);
  if (rc) return rc;
  for (size_t k = 0; k < ids.size(); ++k) {
    if (out[k].status != R3D_RESECT_OK) continue;
    r3d_sfm_data::Pose p;
    std::memcpy(p.R, out[k].rotation, sizeof(p.R));
    std::memcpy(p.C, out[k].center, sizeof(p.C));
    sd->poses[sd->views[ids[k]].id_pose] = p;
  }
  if (n_out) *n_out = (uint32_t)ids.size();
  return R3D_OK;
}

extern "C" int r3d_get_resection_timing(const r3d_ctx* ctx, r3d_resection_timing* out) {
  if (!ctx || !out) return R3D_ERR_INVALID;
  *out = ctx->resection_timing;
  return R3D_OK;
}
