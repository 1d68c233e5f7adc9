// acransac_kernels.cu -- the AC-RANSAC set-up kernels of the filters: matched positions and log-combinatorial tables.
// COMPILED WITH --fmad=false (regard3d_b200/build.py): every double operation below rounds once,
// exactly like the host arithmetic, so discrete decisions are reproducible (see detmath.cuh); k_ac_points's
// s1 * x + c1 must not contract to an FMA.
//   k_ac_points : the putative matches' positions, promoted to double and normalised (the filters' x1 / x2)
//   k_ac_tables : logc_n of every problem (the filters, r3d_relative_poses, r3d_resect_views, r3d_debug_acransac_score)
// The AC-RANSAC itself runs in the persistent kernel of acransac_fused.cu.
#include "acransac.cuh"
#include "detmath.cuh"

namespace r3d {

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
