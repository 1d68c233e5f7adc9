// acransac_kernels.cu -- device side of the a-contrario RANSAC fundamental-matrix filter.
// COMPILED WITH --fmad=false (regard3d_b200/build.py): every double operation below rounds once,
// exactly like the host arithmetic, so discrete decisions are reproducible (see detmath.cuh).
//
// Replaces the per-pair body of ImageCollectionGeometricFilter::Robust_model_estimation(
// GeometricFilter_FMatrix_AC(4.0, 2048), ...) (src/R3DComputeMatches.cpp:2099-2115); upstream
// semantics: SURVEY.md Appendix A.4-A.6.
//   k_f7_solve   : one thread per hypothesis -- 7-point solver (<= 3 models)
//   k_f7_score   : one block per (hypothesis, model) -- M symmetric-epipolar residuals, compaction of
//                  those <= the precision bound, block bitonic sort on (residual, index) in shared
//                  memory, NFA scan, argmin
//   k_f7_inliers : one block per request -- the sorted inlier index list of one model
#include "acransac_device.cuh"

namespace r3d {

// one thread per hypothesis of the essential model: bearings of the 5 sampled matches -> 5-point solver ->
// every E turned into the pixel-space F = K2^-T E K1^-1 the residuals are measured with
__global__ void __launch_bounds__(64) k_e5_solve(const AcPair* __restrict__ pairs, const double2* __restrict__ x1,
                                                 const double2* __restrict__ x2, const AcHyp* __restrict__ hyps,
                                                 uint32_t n_hyp, double* __restrict__ F, uint32_t* __restrict__ nmodels) {
  const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= n_hyp) return;
  const AcHyp hy = hyps[h];
  const AcPair pr = pairs[hy.pair];
  double b1[15], b2[15], Es[90];
  for (int t = 0; t < 5; ++t) {
    const double2 a = x1[pr.pt_ofs + hy.sample[t]];
    const double2 b = x2[pr.pt_ofs + hy.sample[t]];
    bearing(pr.K, a.x, a.y, b1 + 3 * t);
    bearing(pr.K + 3, b.x, b.y, b2 + 3 * t);
  }
  const int nm = fp::five_point(b1, b2, Es);
  nmodels[h] = (uint32_t)nm;
  for (int mi = 0; mi < nm; ++mi) {
    double Fm[9];
    fundamental_from_essential(Es + 9 * mi, pr.K, pr.K + 3, Fm);
    for (int t = 0; t < 9; ++t) F[(size_t)h * 90 + 9 * mi + t] = Fm[t];
  }
}

template <int MODEL>
__global__ void __launch_bounds__(128) k_f7_solve(const AcPair* __restrict__ pairs, const double2* __restrict__ x1,
                                                  const double2* __restrict__ x2, const AcHyp* __restrict__ hyps,
                                                  uint32_t n_hyp, double* __restrict__ F, uint32_t* __restrict__ nmodels) {
  const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= n_hyp) return;
  const AcHyp hy = hyps[h];
  const AcPair pr = pairs[hy.pair];
  double s1[14], s2[14], models[27];
  constexpr int NS = MODEL == 0 ? 7 : 4;
  for (int t = 0; t < NS; ++t) {
    const double2 a = x1[pr.pt_ofs + hy.sample[t]];
    const double2 b = x2[pr.pt_ofs + hy.sample[t]];
    s1[2 * t] = a.x; s1[2 * t + 1] = a.y;
    s2[2 * t] = b.x; s2[2 * t + 1] = b.y;
  }
  const int nm = MODEL == 0 ? seven_point(s1, s2, models) : four_point(s1, s2, models);
  nmodels[h] = (uint32_t)nm;
  for (int t = 0; t < 9 * nm; ++t) F[(size_t)h * (9 * ac_max_models(MODEL)) + t] = models[t];
}

template <int MODEL>
__global__ void __launch_bounds__(256) k_f7_score(const AcPair* __restrict__ pairs, const double2* __restrict__ x1,
                                                  const double2* __restrict__ x2, const AcHyp* __restrict__ hyps,
                                                  const double* __restrict__ F, const uint32_t* __restrict__ nmodels,
                                                  const float* __restrict__ logc_n, const float* __restrict__ logc_k,
                                                  uint32_t cap, AcScore* __restrict__ scores) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ uint32_t s_count;
  __shared__ double s_best_nfa[8];
  __shared__ uint32_t s_best_k[8];
  constexpr uint32_t MAXM = ac_max_models(MODEL);
  const uint32_t h = blockIdx.x / MAXM, mi = blockIdx.x % MAXM;
  if (mi >= nmodels[h]) return;
  const AcHyp hy = hyps[h];
  const AcPair pr = pairs[hy.pair];
  double* se = (double*)smem_raw;
  uint32_t* si = (uint32_t*)(se + cap);
  double Fm[9];
  for (int t = 0; t < 9; ++t) Fm[t] = F[(size_t)h * (9 * MAXM) + 9 * mi + t];
  const uint32_t c = residuals_sorted<MODEL, false>(pr, x1, x2, Fm, se, si, cap, &s_count);
  const NfaBest r = nfa_scan_sorted<MODEL>(pr, se, c, logc_n + pr.tbl_ofs, logc_k, s_best_nfa, s_best_k);
  if (threadIdx.x == 0) {
    AcScore sc;
    sc.nfa = r.nfa;
    sc.err = r.err;
    sc.k = r.k;
    sc.count = s_count;
    scores[(size_t)h * MAXM + mi] = sc;
  }
}

template <int MODEL>
__global__ void __launch_bounds__(256) k_f7_inliers(const AcPair* __restrict__ pairs, const double2* __restrict__ x1,
                                                    const double2* __restrict__ x2, const AcInlierReq* __restrict__ reqs,
                                                    const double* __restrict__ F, uint32_t cap, uint32_t* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ uint32_t s_count;
  const AcInlierReq rq = reqs[blockIdx.x];
  const AcPair pr = pairs[rq.pair];
  double* se = (double*)smem_raw;
  uint32_t* si = (uint32_t*)(se + cap);
  double Fm[9];
  for (int t = 0; t < 9; ++t) Fm[t] = F[(size_t)rq.hyp_model * 9 + t];  // hyp_model = hypothesis * MAX_MODELS + model
  const uint32_t c = residuals_sorted<MODEL, true>(pr, x1, x2, Fm, se, si, cap, &s_count);
  for (uint32_t i = threadIdx.x; i < rq.k && i < c; i += blockDim.x) out[rq.out_ofs + i] = si[i];
}

// ---- positions of the putative matches, promoted to double and normalised exactly like the host would ----
__global__ void __launch_bounds__(256) k_ac_points(const AcPair* __restrict__ pairs, const AcPointSrc* __restrict__ src,
                                                   const uint2* __restrict__ matches, double2* __restrict__ x1,
                                                   double2* __restrict__ x2, uint32_t* __restrict__ bad_flag) {
  const AcPair pr = pairs[blockIdx.y];
  const AcPointSrc ps = src[blockIdx.y];
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < pr.M; k += gridDim.x * blockDim.x) {
    const uint2 m = matches[pr.pt_ofs + k];
    if (m.x >= ps.nI || m.y >= ps.nJ) { atomicExch(bad_flag, 1u); continue; }
    const float2 a = ps.xyI[m.x], b = ps.xyJ[m.y];
    const double xi = (double)a.x, yi = (double)a.y, xj = (double)b.x, yj = (double)b.y;
    x1[pr.pt_ofs + k] = ps.identity ? make_double2(xi, yi) : make_double2(ps.s1 * xi + ps.c1x, ps.s1 * yi + ps.c1y);
    x2[pr.pt_ofs + k] = ps.identity ? make_double2(xj, yj) : make_double2(ps.s2 * xj + ps.c2x, ps.s2 * yj + ps.c2y);
  }
}

// makelogcombi_n (robust_estimator_ACRansac.hpp): logc_n[k] = log10 C(n, k) as a running FLOAT sum over
// i = 1 .. min(k, n - k) of log10(n - i + 1) - log10(i); the partial sums are the entries for smaller k, so one pass per
// pair reproduces the upstream table bit for bit (the log10 table itself comes from the host's libm).
__global__ void __launch_bounds__(128) k_ac_tables(const AcPair* __restrict__ pairs, uint32_t n_pairs, const float* __restrict__ vlog10,
                                                   float* __restrict__ logc_n) {
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n_pairs) return;
  const uint32_t n = pairs[a].M;
  float* t = logc_n + pairs[a].tbl_ofs;
  t[0] = 0.f;
  float r = 0.f;
  // t[n + 1] = a bound on |t[k] - log10 C(n, k)| for every k: each step rounds the difference and the running sum
  // (half an ulp of each) and reads two table entries that are within an ulp of the true logarithms
  double err = 0.0;
  for (uint32_t i = 1; i <= n / 2; ++i) {
    const float d = __fsub_rn(vlog10[n - i + 1], vlog10[i]);
    r = __fadd_rn(r, d);
    t[i] = r;
    err += 5.97e-8 * ((double)fabsf(r) + (double)fabsf(d)) + 1.2e-7 * ((double)vlog10[n - i + 1] + (double)vlog10[i]);
  }
  for (uint32_t k = n / 2 + 1; k <= n; ++k) t[k] = (k >= n) ? 0.f : t[n - k];
  t[n + 1] = (float)(err * 1.001 + 1e-6);
}

int launch_ac_tables(r3d_ctx* ctx, DeviceWorker& w, const AcPair* pairs, uint32_t n_pairs, const float* vlog10, float* logc_n) {
  if (!n_pairs) return R3D_OK;
  k_ac_tables<<<(n_pairs + 127) / 128, 128, 0, w.stream>>>(pairs, n_pairs, vlog10, logc_n);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_ac_points(r3d_ctx* ctx, DeviceWorker& w, const AcPair* pairs, const AcPointSrc* src, uint32_t n_pairs,
                     const uint2* matches, double2* x1, double2* x2, uint32_t* bad_flag) {
  if (!n_pairs) return R3D_OK;
  for (uint32_t p0 = 0; p0 < n_pairs; p0 += 65535u) {  // gridDim.y limit
    const uint32_t np = std::min(65535u, n_pairs - p0);
    k_ac_points<<<dim3(8, np), 256, 0, w.stream>>>(pairs + p0, src + p0, matches, x1, x2, bad_flag);
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

// ------------------------------------------------------------------------------------------------
int launch_f7_solve(r3d_ctx* ctx, DeviceWorker& w, int model, const AcPair* pairs, const double2* x1, const double2* x2,
                    const AcHyp* hyps, uint32_t n_hyp, double* F, uint32_t* nmodels) {
  if (!n_hyp) return R3D_OK;
  if (model == 0) k_f7_solve<0><<<(n_hyp + 127) / 128, 128, 0, w.stream>>>(pairs, x1, x2, hyps, n_hyp, F, nmodels);
  else if (model == 1) k_f7_solve<1><<<(n_hyp + 127) / 128, 128, 0, w.stream>>>(pairs, x1, x2, hyps, n_hyp, F, nmodels);
  else k_e5_solve<<<(n_hyp + 63) / 64, 64, 0, w.stream>>>(pairs, x1, x2, hyps, n_hyp, F, nmodels);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_f7_score(r3d_ctx* ctx, DeviceWorker& w, int model, const AcPair* pairs, const double2* x1, const double2* x2,
                    const AcHyp* hyps, uint32_t n_hyp, const double* F, const uint32_t* nmodels, const float* logc_n,
                    const float* logc_k, uint32_t cap, AcScore* scores) {
  if (!n_hyp) return R3D_OK;
  const size_t smem = (size_t)cap * 12;
  if (model == 0) {
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_f7_score<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_f7_score<0><<<n_hyp * 3, 256, smem, w.stream>>>(pairs, x1, x2, hyps, F, nmodels, logc_n, logc_k, cap, scores);
  } else if (model == 1) {
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_f7_score<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_f7_score<1><<<n_hyp * 1, 256, smem, w.stream>>>(pairs, x1, x2, hyps, F, nmodels, logc_n, logc_k, cap, scores);
  } else {
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_f7_score<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_f7_score<2><<<n_hyp * 10, 256, smem, w.stream>>>(pairs, x1, x2, hyps, F, nmodels, logc_n, logc_k, cap, scores);
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_f7_inliers(r3d_ctx* ctx, DeviceWorker& w, int model, const AcPair* pairs, const double2* x1, const double2* x2,
                      const AcInlierReq* reqs, uint32_t n_req, const double* F, uint32_t cap, uint32_t* out) {
  if (!n_req) return R3D_OK;
  const size_t smem = (size_t)cap * 12;
  if (model == 0) {
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_f7_inliers<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_f7_inliers<0><<<n_req, 256, smem, w.stream>>>(pairs, x1, x2, reqs, F, cap, out);
  } else if (model == 1) {
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_f7_inliers<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_f7_inliers<1><<<n_req, 256, smem, w.stream>>>(pairs, x1, x2, reqs, F, cap, out);
  } else {
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_f7_inliers<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_f7_inliers<2><<<n_req, 256, smem, w.stream>>>(pairs, x1, x2, reqs, F, cap, out);
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

}  // namespace r3d

// ---- r3d_debug_detmath: the deterministic transcendentals on the device and in this translation unit's host code ----
namespace r3d {
namespace {

R3D_HD double detmath_eval(int fn, double x) {
  return fn == 0 ? dm::log10_det(x) : fn == 1 ? dm::cbrt_det(x) : fn == 2 ? dm::cos_det(x) : dm::acos_det(x);
}

__global__ void k_debug_detmath(int fn, const double* __restrict__ x, uint64_t n, double* __restrict__ y) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    y[i] = detmath_eval(fn, x[i]);
}

}  // namespace
}  // namespace r3d

extern "C" int r3d_debug_detmath(int fn, int on_device, const double* x, uint64_t n, double* y) {
  if (fn < 0 || fn > 3 || (n && (!x || !y))) return r3d::fail(nullptr, R3D_ERR_INVALID, "r3d_debug_detmath: bad arguments");
  if (!on_device) {
    for (uint64_t i = 0; i < n; ++i) y[i] = r3d::detmath_eval(fn, x[i]);
    return R3D_OK;
  }
  if (!n) return R3D_OK;
  double* d = nullptr;
  cudaError_t e = cudaMalloc(&d, 2 * n * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(d, x, n * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    r3d::k_debug_detmath<<<(unsigned)std::min<uint64_t>((n + 255) / 256, 4096), 256>>>(fn, d, n, d + n);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(y, d + n, n * sizeof(double), cudaMemcpyDeviceToHost);
  if (d) cudaFree(d);
  return e == cudaSuccess ? R3D_OK : r3d::fail(nullptr, R3D_ERR_CUDA, std::string("r3d_debug_detmath: ") + cudaGetErrorString(e));
}
