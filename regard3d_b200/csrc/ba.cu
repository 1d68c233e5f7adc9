// ba.cu -- bundle adjustment on the GPU: Levenberg-Marquardt with a point Schur complement.
//
// Replaces openMVG::sfm::Bundle_Adjustment_Ceres::Adjust as reached from the SfM engines' Process()
// (src/threads/R3DTriangulationThread.cpp:441, :512, :250); algorithm restated in SURVEY.md A.7 and
// mirrored by oracle/oracle_ba.cpp (Ceres' trust-region LM, Jacobi scaling, Huber corrector,
// SPARSE_SCHUR).  Everything is FP64.  Per LM iteration:
//   k_ba_eval      one thread per observation: residual, analytic Jacobian, Huber corrector ->
//                  gradient and diag(J^T J) (atomics), cost (block reduction)
//   k_ba_schur     one WARP per 3-D point: stages the point's observation Jacobians in shared memory,
//                  V = sum Jp^T Jp + D^2 (warp-shuffle reduction), V^-1, then the block pairs
//                  S[a,b] -= W_a V^-1 W_b^T and rhs[a] += W_a V^-1 g_p are spread over the lanes
//                  (atomicAdd into the dense reduced camera system, upper-triangular block form;
//                  the intrinsic-intrinsic block is pre-reduced per CTA in shared memory)
//   k_chol_*       blocked dense Cholesky of the reduced system + triangular solves
//   k_ba_backsub   one thread per point: delta_p = V^-1 (-g_p - W^T delta_B)
//   k_ba_update    x + scale*delta -> candidate parameters, ||dx||, ||x||, model cost change
//   k_ba_cost      cost at the candidate
// The Jacobian is recomputed where it is needed (300 flop per observation) instead of being stored:
// the path is bound by the observation stream, not by arithmetic.
#include "r3d_internal.cuh"
#include "ba_model.cuh"
#include "lm_trust_region.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>

namespace cg = cooperative_groups;

namespace r3d {
namespace ba {

constexpr int kObsDoubles = 12 + 12 + 6 + 2;  // Jc, Jg, Jp, r

struct Dev {
  uint32_t n_cams, n_pts, n_intr, nB, refine_intr;
  uint32_t owns_shared;                    // multi-rank: 1 on the rank that counts the replicated camera/intrinsic
                                           // parameters in the step norms and the model cost change
  uint64_t n_obs;
  double huber_a;
  double *poses, *intr, *pts;              // current parameters
  double *poses_new, *intr_new, *pts_new;  // candidate
  const uint32_t *obs_cam, *obs_pt, *cam_intr;
  const double2* obs_xy;
  const uint32_t *pt_ofs, *pt_obs;         // point -> observation CSR
  double *scale, *gu, *du, *g, *diag, *delta;  // nparam each (u = unscaled accumulators)
  double *S, *rhs, *Vinv;
  const uint8_t* intr_model;               // per group: openMVG EINTRINSIC 1..5 (nullptr: all radial K3)
  const double* intr_ext;                  // per group 2 doubles: Brown t1 t2 / fisheye k4 (nullptr: zeros); held fixed
  uint32_t n_priors;                       // pose-centre priors (ViewPriors): camera, centre, weight
  const uint32_t* prior_cam;
  const double *prior_center, *prior_weight;
  double prior_huber_a;
  double* scal;                            // [0] cost [1] model_cost_change*2 [2] |dx|^2 [3] |x|^2 [4] not-PD flag
};

__device__ __forceinline__ uint32_t intr_col(const Dev& d, uint32_t g) { return 6 * d.n_cams + 6 * g; }
__device__ __forceinline__ int model_of(const Dev& d, uint32_t g) { return d.intr_model ? (int)d.intr_model[g] : 3; }
__device__ __forceinline__ const double* ext_of(const Dev& d, uint32_t g) { return d.intr_ext ? d.intr_ext + 2 * (size_t)g : nullptr; }

__device__ __forceinline__ double block_sum(double v, double* smem) {
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0;
  if (threadIdx.x < 32) {
    t = (threadIdx.x < (blockDim.x >> 5)) ? smem[threadIdx.x] : 0.0;
    for (int o = 16; o >= 1; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  __syncthreads();
  return t;  // valid in thread 0
}

// ---- cost only ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ba_cost(Dev d, const double* poses, const double* intr, const double* pts,
                                                 double* out_cost) {
  __shared__ double sm[8];
  double c = 0;
  for (uint64_t o = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; o < d.n_obs; o += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t cam = d.obs_cam[o], pt = d.obs_pt[o];
    const double2 xy = d.obs_xy[o];
    double r[2];
    const uint32_t gi = d.cam_intr[cam];
    residual_only(model_of(d, gi), intr + 6 * (size_t)gi, ext_of(d, gi), poses + 6 * (size_t)cam, pts + 3 * (size_t)pt, xy.x, xy.y, r);
    double rho1;
    c += 0.5 * huber_rho(r[0] * r[0] + r[1] * r[1], d.huber_a, &rho1);
  }
  c = block_sum(c, sm);
  if (threadIdx.x == 0) atomicAdd(out_cost, c);
}

// |residual| per coordinate (OpenMVGHelper::calculateResiduals)
__global__ void __launch_bounds__(256) k_ba_abs_residuals(Dev d, double* res) {
  for (uint64_t o = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; o < d.n_obs; o += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t cam = d.obs_cam[o], pt = d.obs_pt[o];
    const double2 xy = d.obs_xy[o];
    double r[2];
    const uint32_t gi = d.cam_intr[cam];
    residual_only(model_of(d, gi), d.intr + 6 * (size_t)gi, ext_of(d, gi), d.poses + 6 * (size_t)cam, d.pts + 3 * (size_t)pt, xy.x, xy.y, r);
    res[2 * o] = fabs(r[0]);
    res[2 * o + 1] = fabs(r[1]);
  }
}

// ---- gradient + diag(J^T J), unscaled ----------------------------------------------------------
__global__ void __launch_bounds__(256) k_ba_eval(Dev d) {
  for (uint64_t o = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; o < d.n_obs; o += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t cam = d.obs_cam[o], pt = d.obs_pt[o], gi = d.cam_intr[cam];
    const double2 xy = d.obs_xy[o];
    double r[2], Ji[12], Jc[12], Jp[6];
    residual_jacobian(model_of(d, gi), d.intr + 6 * (size_t)gi, ext_of(d, gi), d.poses + 6 * (size_t)cam, d.pts + 3 * (size_t)pt,
                      xy.x, xy.y, r, Ji, Jc, Jp);
    double rho1;
    huber_rho(r[0] * r[0] + r[1] * r[1], d.huber_a, &rho1);
    // Corrector (rho'' <= 0): residual and Jacobian scaled by sqrt(rho') -> J^T r and J^T J scale by rho'
    for (int k = 0; k < 6; ++k) {
      atomicAdd(&d.gu[6 * (size_t)cam + k], rho1 * (Jc[k] * r[0] + Jc[6 + k] * r[1]));
      atomicAdd(&d.du[6 * (size_t)cam + k], rho1 * (Jc[k] * Jc[k] + Jc[6 + k] * Jc[6 + k]));
    }
    if (d.refine_intr) {
      // every observation of a group hits the same 12 addresses: reduce over the warp first when the
      // active lanes agree on the group (always true for a single shared intrinsic)
      const unsigned active = __activemask();
      const bool uniform = __match_any_sync(active, gi) == active;
      for (int k = 0; k < 6; ++k) {
        double gv = rho1 * (Ji[k] * r[0] + Ji[6 + k] * r[1]);
        double dv = rho1 * (Ji[k] * Ji[k] + Ji[6 + k] * Ji[6 + k]);
        if (uniform && active == 0xffffffffu) {
          for (int o = 16; o >= 1; o >>= 1) {
            gv += __shfl_xor_sync(0xffffffffu, gv, o);
            dv += __shfl_xor_sync(0xffffffffu, dv, o);
          }
          if ((threadIdx.x & 31) == 0) {
            atomicAdd(&d.gu[intr_col(d, gi) + k], gv);
            atomicAdd(&d.du[intr_col(d, gi) + k], dv);
          }
        } else {
          atomicAdd(&d.gu[intr_col(d, gi) + k], gv);
          atomicAdd(&d.du[intr_col(d, gi) + k], dv);
        }
      }
    }
    for (int k = 0; k < 3; ++k) {
      atomicAdd(&d.gu[(size_t)d.nB + 3 * (size_t)pt + k], rho1 * (Jp[k] * r[0] + Jp[3 + k] * r[1]));
      atomicAdd(&d.du[(size_t)d.nB + 3 * (size_t)pt + k], rho1 * (Jp[k] * Jp[k] + Jp[3 + k] * Jp[3 + k]));
    }
  }
}

__global__ void k_ba_make_scale(double* scale, const double* du, size_t n) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < n) scale[j] = 1.0 / (1.0 + sqrt(du[j]));  // Ceres Jacobi scaling: 1 / (1 + ||column||)
}
__global__ void k_ba_apply_scale(const double* scale, const double* gu, const double* du, double* g, double* diag, size_t n,
                                 double* gmax) {
  __shared__ double sm[8];
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  double m = 0;
  if (j < n) {
    g[j] = gu[j] * scale[j];
    diag[j] = du[j] * scale[j] * scale[j];
    m = fabs(gu[j]);  // unscaled gradient for the gradient tolerance
  }
  for (int o = 16; o >= 1; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, sm[w]);
    // non-negative doubles order like their bit patterns
    atomicMax((unsigned long long*)gmax, (unsigned long long)__double_as_longlong(m));
  }
}

// scaled, corrected Jacobian blocks of one observation
__device__ __forceinline__ void scaled_jacobian(const Dev& d, uint32_t o, double* Jc, double* Jg, double* Jp, double* r,
                                                uint32_t* colc, int* colg) {
  const uint32_t cam = d.obs_cam[o], pt = d.obs_pt[o], gi = d.cam_intr[cam];
  const double2 xy = d.obs_xy[o];
  double Ji[12];
  residual_jacobian(model_of(d, gi), d.intr + 6 * (size_t)gi, ext_of(d, gi), d.poses + 6 * (size_t)cam, d.pts + 3 * (size_t)pt, xy.x,
                    xy.y, r, Ji, Jc, Jp);
  double rho1;
  huber_rho(r[0] * r[0] + r[1] * r[1], d.huber_a, &rho1);
  const double sq = sqrt(rho1);
  r[0] *= sq; r[1] *= sq;
  const double* sc = d.scale + 6 * (size_t)cam;
  const double* sp = d.scale + (size_t)d.nB + 3 * (size_t)pt;
  for (int a = 0; a < 2; ++a) {
    for (int k = 0; k < 6; ++k) Jc[6 * a + k] *= sq * sc[k];
    for (int k = 0; k < 3; ++k) Jp[3 * a + k] *= sq * sp[k];
  }
  *colc = 6 * cam;
  if (d.refine_intr) {
    const double* sg = d.scale + intr_col(d, gi);
    for (int a = 0; a < 2; ++a)
      for (int k = 0; k < 6; ++k) Jg[6 * a + k] = Ji[6 * a + k] * sq * sg[k];
    *colg = (int)intr_col(d, gi);
  } else {
    for (int k = 0; k < 12; ++k) Jg[k] = 0.0;
    *colg = -1;
  }
}

__device__ __forceinline__ void inv3_sym(const double* V, double* Vi) {
  const double c00 = V[4] * V[8] - V[5] * V[7], c01 = V[5] * V[6] - V[3] * V[8], c02 = V[3] * V[7] - V[4] * V[6];
  const double det = V[0] * c00 + V[1] * c01 + V[2] * c02;
  Vi[0] = c00 / det; Vi[1] = (V[2] * V[7] - V[1] * V[8]) / det; Vi[2] = (V[1] * V[5] - V[2] * V[4]) / det;
  Vi[3] = c01 / det; Vi[4] = (V[0] * V[8] - V[2] * V[6]) / det; Vi[5] = (V[2] * V[3] - V[0] * V[5]) / det;
  Vi[6] = c02 / det; Vi[7] = (V[1] * V[6] - V[0] * V[7]) / det; Vi[8] = (V[0] * V[4] - V[1] * V[3]) / det;
}

// add the 6x6 block `blk` (row-major) at block position (ca, cb) of the upper-triangular block form
__device__ __forceinline__ void add_block_upper(double* S, uint32_t nB, uint32_t ca, uint32_t cb, const double* blk, double sign) {
  if (ca <= cb) {
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) atomicAdd(&S[(size_t)(ca + i) * nB + cb + j], sign * blk[6 * i + j]);
  } else {  // store the transpose at (cb, ca)
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) atomicAdd(&S[(size_t)(cb + j) * nB + ca + i], sign * blk[6 * i + j]);
  }
}

// ---- Schur complement: one CTA per point, any track length (the general path) ---------------------------
// Points the batched kernel below cannot take (more than 32 observations -- real tracks span hundreds of views --,
// more than 2 intrinsic groups, a camera that sees the point twice) are listed and handled here: the scaled Jacobians
// and W blocks of the point's observations are staged in a per-CTA slice of GLOBAL scratch (`cap` observations), so
// there is no limit on the track length (round 1 staged them in shared memory and returned R3D_ERR_UNSUPPORTED beyond
// 64).  Same algebra as the batched kernel: V = sum Jp^T Jp + D^2, W_c = Jc^T Jp per camera, W_g = sum over the
// observations of an intrinsic group, S -= W_a V^-1 W_b^T over all entry pairs, U terms added directly.
constexpr int kCtaThreads = 128;
__global__ void __launch_bounds__(kCtaThreads) k_ba_schur_cta(Dev d, const uint32_t* __restrict__ list, uint32_t n_list,
                                                              double inv_radius, double* __restrict__ scratch,
                                                              int* __restrict__ cols, uint32_t cap) {
  __shared__ double s_red[6][kCtaThreads / 32];
  __shared__ double s_Vi[9], s_Vg[3];
  double* J = scratch + (size_t)blockIdx.x * cap * (kObsDoubles + 36);
  double* W = J + (size_t)cap * kObsDoubles;
  int* colc = cols + (size_t)blockIdx.x * cap * 3;
  int* colg = colc + cap;
  int* lead = colg + cap;
  const int tid = threadIdx.x;
  for (uint32_t li = blockIdx.x; li < n_list; li += gridDim.x) {
    const uint32_t ip = list[li];
    const uint32_t b = d.pt_ofs[ip], e = d.pt_ofs[ip + 1];
    const int nobs = (int)(e - b);
    __syncthreads();  // the previous point's readers are done with the scratch slice
    // 1. stage the scaled Jacobians of this point's observations
    for (int t = tid; t < nobs; t += kCtaThreads) {
      double* jt = J + (size_t)t * kObsDoubles;
      uint32_t cc;
      int cg;
      scaled_jacobian(d, d.pt_obs[b + t], jt, jt + 12, jt + 24, jt + 30, &cc, &cg);
      colc[t] = (int)cc;
      colg[t] = cg;
    }
    __syncthreads();
    // 2. V = sum Jp^T Jp + D^2, V^-1, V^-1 g_p
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (int t = tid; t < nobs; t += kCtaThreads) {
      const double* jp = J + (size_t)t * kObsDoubles + 24;
      v[0] += jp[0] * jp[0] + jp[3] * jp[3]; v[1] += jp[0] * jp[1] + jp[3] * jp[4]; v[2] += jp[0] * jp[2] + jp[3] * jp[5];
      v[3] += jp[1] * jp[1] + jp[4] * jp[4]; v[4] += jp[1] * jp[2] + jp[4] * jp[5]; v[5] += jp[2] * jp[2] + jp[5] * jp[5];
    }
    for (int k = 0; k < 6; ++k) {
      for (int o = 16; o >= 1; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
      if ((tid & 31) == 0) s_red[k][tid >> 5] = v[k];
    }
    __syncthreads();
    const size_t pcol = (size_t)d.nB + 3 * (size_t)ip;
    if (tid == 0) {
      double vv[6];
      for (int k = 0; k < 6; ++k) {
        vv[k] = 0.0;
        for (int wv = 0; wv < kCtaThreads / 32; ++wv) vv[k] += s_red[k][wv];
      }
      double V[9] = {vv[0], vv[1], vv[2], vv[1], vv[3], vv[4], vv[2], vv[4], vv[5]};
      for (int i = 0; i < 3; ++i) V[4 * i] += fmin(fmax(d.diag[pcol + i], 1e-6), 1e32) * inv_radius;
      double Vi[9];
      inv3_sym(V, Vi);
      for (int i = 0; i < 9; ++i) { d.Vinv[9 * (size_t)ip + i] = Vi[i]; s_Vi[i] = Vi[i]; }
      const double gp[3] = {d.g[pcol], d.g[pcol + 1], d.g[pcol + 2]};
      for (int i = 0; i < 3; ++i) s_Vg[i] = Vi[3 * i] * gp[0] + Vi[3 * i + 1] * gp[1] + Vi[3 * i + 2] * gp[2];
    }
    __syncthreads();
    double Vi[9], Vg[3];
    for (int i = 0; i < 9; ++i) Vi[i] = s_Vi[i];
    for (int i = 0; i < 3; ++i) Vg[i] = s_Vg[i];
    // 3. W blocks (6x3) of every observation's camera and intrinsic group; the U part of S
    for (int t = tid; t < nobs; t += kCtaThreads) {
      const double* jt = J + (size_t)t * kObsDoubles;
      const double *jc = jt, *jg = jt + 12, *jp = jt + 24;
      double* wc = W + (size_t)t * 36;
      double* wg = wc + 18;
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 3; ++j) {
          wc[3 * i + j] = jc[i] * jp[j] + jc[6 + i] * jp[3 + j];
          wg[3 * i + j] = jg[i] * jp[j] + jg[6 + i] * jp[3 + j];
        }
      double blk[36];
      const uint32_t cc = (uint32_t)colc[t];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) blk[6 * i + j] = jc[i] * jc[j] + jc[6 + i] * jc[6 + j];
      add_block_upper(d.S, d.nB, cc, cc, blk, 1.0);
      const int cg = colg[t];
      if (cg >= 0) {
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j < 6; ++j) blk[6 * i + j] = jc[i] * jg[j] + jc[6 + i] * jg[6 + j];
        add_block_upper(d.S, d.nB, cc, (uint32_t)cg, blk, 1.0);
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j < 6; ++j) blk[6 * i + j] = jg[i] * jg[j] + jg[6 + i] * jg[6 + j];
        add_block_upper(d.S, d.nB, (uint32_t)cg, (uint32_t)cg, blk, 1.0);
      }
      // the first observation of each intrinsic group leads it
      int ld = t;
      if (cg >= 0)
        for (int u = 0; u < t; ++u)
          if (colg[u] == cg) { ld = u; break; }
      lead[t] = ld;
    }
    __syncthreads();
    // merge the group blocks into their leaders (W_g = sum over the group's observations), retire the others
    for (int t = tid; t < nobs; t += kCtaThreads) {
      if (colg[t] >= 0 && lead[t] != t) {
        double* wl = W + (size_t)lead[t] * 36 + 18;
        const double* wt = W + (size_t)t * 36 + 18;
        for (int q = 0; q < 18; ++q) atomicAdd(&wl[q], wt[q]);
      }
    }
    __syncthreads();
    for (int t = tid; t < nobs; t += kCtaThreads)
      if (colg[t] >= 0 && lead[t] != t) colg[t] = -1;
    __syncthreads();
    // 4. Schur part over the 2 * nobs entries (camera t -> entry 2t, group t -> entry 2t + 1; merged groups are -1)
    const long long nblk = 2LL * nobs;
    for (long long a = tid; a < nblk; a += kCtaThreads) {  // rhs[a] += W_a V^-1 g_p
      const int ca = (a & 1) ? colg[a >> 1] : colc[a >> 1];
      if (ca < 0) continue;
      const double* wa = W + (size_t)(a >> 1) * 36 + (a & 1) * 18;
      for (int i = 0; i < 6; ++i) atomicAdd(&d.rhs[ca + i], wa[3 * i] * Vg[0] + wa[3 * i + 1] * Vg[1] + wa[3 * i + 2] * Vg[2]);
    }
    const long long npairs = nblk * (nblk + 1) / 2;
    for (long long pr = tid; pr < npairs; pr += kCtaThreads) {
      long long hi = (long long)((sqrt(8.0 * (double)pr + 1.0) - 1.0) * 0.5);
      while ((hi + 1) * (hi + 2) / 2 <= pr) ++hi;
      while (hi * (hi + 1) / 2 > pr) --hi;
      const long long lo = pr - hi * (hi + 1) / 2;  // lo <= hi
      const int ch = (hi & 1) ? colg[hi >> 1] : colc[hi >> 1];
      const int cl = (lo & 1) ? colg[lo >> 1] : colc[lo >> 1];
      if (ch < 0 || cl < 0) continue;
      const double* wl = W + (size_t)(lo >> 1) * 36 + (lo & 1) * 18;
      const double* wh = W + (size_t)(hi >> 1) * 36 + (hi & 1) * 18;
      double WV[18];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 3; ++j) WV[3 * i + j] = wl[3 * i] * Vi[j] + wl[3 * i + 1] * Vi[3 + j] + wl[3 * i + 2] * Vi[6 + j];
      double blk[36];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) blk[6 * i + j] = WV[3 * i] * wh[3 * j] + WV[3 * i + 1] * wh[3 * j + 1] + WV[3 * i + 2] * wh[3 * j + 2];
      // blk = W_lo V^-1 W_hi^T contributes to S[cl, ch]; for lo != hi the mirrored term S[ch, cl] is its transpose: in
      // upper-block form both land on the same stored block (so a block shared by two different entries gets blk + blk^T)
      if (lo != hi && cl == ch) {
        double sym[36];
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j < 6; ++j) sym[6 * i + j] = blk[6 * i + j] + blk[6 * j + i];
        add_block_upper(d.S, d.nB, (uint32_t)cl, (uint32_t)ch, sym, -1.0);
      } else {
        add_block_upper(d.S, d.nB, (uint32_t)cl, (uint32_t)ch, blk, -1.0);
      }
    }
  }
}

// ---- Schur complement, batched and atomic-free inside a CTA (the default path) --------------------------
// The warp-per-point kernel above spends its time in ~1 100 fp64 global atomics per point.  Here a CTA takes a
// BATCH of consecutive points of a camera-sorted processing order (host: setup_problem), so that the batch touches
// only a few distinct 6-wide blocks of S (its cameras + intrinsic groups):
//   stage 1  warp per point, lane per observation: scaled Jacobians, V^-1, and one shared-memory ENTRY per block
//            of the point: W (6x3), W V^-1, W V^-1 g_p, and for camera entries Jc, Jg (the U terms)
//   stage 2  OUTPUT-centric: 36 threads own one 6x6 block pair (lo, hi) of the batch's local block table, walk the
//            batch's points and accumulate  [U term] - (W_lo V^-1) W_hi^T  in a register; 6 threads own a block's
//            right-hand side.  No atomics, no conflicts.
//   flush    one global atomicAdd per non-zero output: a few thousand per batch instead of ~1 100 per POINT.
// Limits of this path (else the host selects the per-point kernel): <= kBatchEntries entries and <= kBatchBlocks
// distinct blocks per batch, <= 32 observations and <= 2 intrinsic groups per point, no point observed twice by
// one camera.
constexpr int kBatchPoints = 24;    // points per CTA batch (upper bound; the host cuts batches)
constexpr int kBatchEntries = 144;  // entries per batch
constexpr int kBatchBlocks = 40;    // distinct 6-wide blocks per batch
constexpr int kEntryDoubles = 72;   // W 18 | WV 18 | WVg 6 | Jc 12 | Jg 12 | Jp 6
constexpr size_t kBatchSmemBytes = ((size_t)kBatchEntries * kEntryDoubles + (size_t)kBatchPoints * 2 * 36) * sizeof(double);
// Static structure of a batch, built once per problem on the host (setup_problem): the processing order, the
// first entry of every ordered point (entries of a point: its observations in CSR order, then its distinct
// intrinsic groups in order of first appearance), the batch's sorted distinct block columns and every entry's
// index into them.
struct BatchDesc { uint32_t first, count, ent_first, nblk; };
struct BatchTables {
  const BatchDesc* batches;
  const uint32_t* pt_order;    // [n_pts]
  const uint32_t* ent_start;   // [n_pts + 1] by ordered position
  const int* cols;             // [n_batches][kBatchBlocks]
  const unsigned char* lblk;   // [total entries]
};

__global__ void __launch_bounds__(256, 2) k_ba_schur_batched(Dev d, BatchTables bt, double inv_radius) {
  extern __shared__ __align__(16) double bsm[];
  double* ent = bsm;                                            // [kBatchEntries][kEntryDoubles]
  double* gg = ent + (size_t)kBatchEntries * kEntryDoubles;      // [kBatchPoints * 2][36]  sum Jg^T Jg of the group entries
  __shared__ int s_col[kBatchBlocks];                            // local block -> first column in S
  __shared__ unsigned char s_lblk[kBatchEntries];                // per entry: local block
  __shared__ int s_ggidx[kBatchEntries];                         // group entries: GG slot ; camera entries: -2 - (own group column, -1 if none)
  __shared__ unsigned char s_slot[kBatchPoints][kBatchBlocks];   // entry of (point, local block), 255 = absent
  __shared__ uint32_t s_pent[kBatchPoints + 1];                  // first entry of each point, relative to the batch
  const BatchDesc bd = bt.batches[blockIdx.x];
  const uint32_t* pt_order = bt.pt_order;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int P = (int)bd.count;
  const int L = (int)bd.nblk;
  for (int k = threadIdx.x; k <= P; k += blockDim.x) s_pent[k] = bt.ent_start[bd.first + k] - bd.ent_first;
  for (int k = threadIdx.x; k < L; k += blockDim.x) s_col[k] = bt.cols[(size_t)blockIdx.x * kBatchBlocks + k];
  for (int k = threadIdx.x; k < kBatchPoints * kBatchBlocks; k += blockDim.x) ((unsigned char*)s_slot)[k] = 255;
  __syncthreads();
  const int nent = (int)s_pent[P];
  for (int q = threadIdx.x; q < nent; q += blockDim.x) s_lblk[q] = bt.lblk[bd.ent_first + q];
  // ---- stage 1: warp per point ----
  for (int k = warp; k < P; k += 8) {
    const uint32_t ip = pt_order[bd.first + k];
    const uint32_t b = d.pt_ofs[ip], e = d.pt_ofs[ip + 1];
    const int nobs = (int)(e - b);
    const uint32_t e0 = s_pent[k];
    double Jc[12], Jg[12], Jp[6], r[2];
    uint32_t colc = 0;
    int colg = -1;
    const bool has = lane < nobs;
    if (has) scaled_jacobian(d, d.pt_obs[b + lane], Jc, Jg, Jp, r, &colc, &colg);
    else {
      for (int i = 0; i < 6; ++i) Jp[i] = 0.0;
    }
    double v[6] = {Jp[0] * Jp[0] + Jp[3] * Jp[3], Jp[0] * Jp[1] + Jp[3] * Jp[4], Jp[0] * Jp[2] + Jp[3] * Jp[5],
                   Jp[1] * Jp[1] + Jp[4] * Jp[4], Jp[1] * Jp[2] + Jp[4] * Jp[5], Jp[2] * Jp[2] + Jp[5] * Jp[5]};
    for (int q = 0; q < 6; ++q)
      for (int o = 16; o >= 1; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
    const size_t pcol = (size_t)d.nB + 3 * (size_t)ip;
    double V[9] = {v[0], v[1], v[2], v[1], v[3], v[4], v[2], v[4], v[5]};
    for (int i = 0; i < 3; ++i) V[4 * i] += fmin(fmax(d.diag[pcol + i], 1e-6), 1e32) * inv_radius;
    double Vi[9];
    inv3_sym(V, Vi);
    if (lane == 0)
      for (int i = 0; i < 9; ++i) d.Vinv[9 * (size_t)ip + i] = Vi[i];
    const double gp[3] = {d.g[pcol], d.g[pcol + 1], d.g[pcol + 2]};
    const double Vg[3] = {Vi[0] * gp[0] + Vi[1] * gp[1] + Vi[2] * gp[2], Vi[3] * gp[0] + Vi[4] * gp[1] + Vi[5] * gp[2],
                          Vi[6] * gp[0] + Vi[7] * gp[1] + Vi[8] * gp[2]};
    if (has) {  // camera entry of observation `lane`
      double* en = ent + (size_t)(e0 + lane) * kEntryDoubles;
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        double w3[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          w3[j] = Jc[i] * Jp[j] + Jc[6 + i] * Jp[3 + j];
          en[3 * i + j] = w3[j];
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) en[18 + 3 * i + j] = w3[0] * Vi[j] + w3[1] * Vi[3 + j] + w3[2] * Vi[6 + j];
        en[36 + i] = w3[0] * Vg[0] + w3[1] * Vg[1] + w3[2] * Vg[2];
      }
#pragma unroll
      for (int q = 0; q < 12; ++q) { en[42 + q] = Jc[q]; en[54 + q] = Jg[q]; }
#pragma unroll
      for (int q = 0; q < 6; ++q) en[66 + q] = Jp[q];
      s_ggidx[e0 + lane] = -2 - colg;
    }
    __syncwarp();
    // group entries (<= 2 distinct groups per point): W_g = sum_t Jg_t^T Jp_t and GG = sum_t Jg_t^T Jg_t over the
    // observations of the group, ONE output element per lane, reading the camera entries just written
    if (d.refine_intr) {
      unsigned todo = __ballot_sync(0xffffffffu, has);
      int gslot = 0;
      while (todo) {
        const int leader = __ffs(todo) - 1;
        const int gcol = __shfl_sync(0xffffffffu, colg, leader);
        todo &= ~__ballot_sync(0xffffffffu, has && colg == gcol);
        double* en = ent + (size_t)(e0 + nobs + gslot) * kEntryDoubles;
        double* G = gg + (size_t)(2 * k + gslot) * 36;
        for (int q = lane; q < 54; q += 32) {  // 18 elements of W_g, then 36 of GG
          double acc = 0.0;
          if (q < 18) {
            const int i = q / 3, j = q % 3;
            for (int t = 0; t < nobs; ++t) {
              if (s_ggidx[e0 + t] != -2 - gcol) continue;
              const double* et = ent + (size_t)(e0 + t) * kEntryDoubles;
              acc += et[54 + i] * et[66 + j] + et[60 + i] * et[69 + j];
            }
            en[q] = acc;
          } else {
            const int i = (q - 18) / 6, j = (q - 18) % 6;
            for (int t = 0; t < nobs; ++t) {
              if (s_ggidx[e0 + t] != -2 - gcol) continue;
              const double* et = ent + (size_t)(e0 + t) * kEntryDoubles;
              acc += et[54 + i] * et[54 + j] + et[60 + i] * et[60 + j];
            }
            G[q - 18] = acc;
          }
        }
        __syncwarp();
        if (lane < 6) {  // WV and WVg of the merged group block
          const int i = lane;
          const double w0 = en[3 * i], w1 = en[3 * i + 1], w2 = en[3 * i + 2];
          for (int j = 0; j < 3; ++j) en[18 + 3 * i + j] = w0 * Vi[j] + w1 * Vi[3 + j] + w2 * Vi[6 + j];
          en[36 + i] = w0 * Vg[0] + w1 * Vg[1] + w2 * Vg[2];
        }
        if (lane == 0) s_ggidx[e0 + nobs + gslot] = 2 * k + gslot;
        ++gslot;
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < P; k += blockDim.x)
    for (uint32_t q = s_pent[k]; q < s_pent[k + 1]; ++q) s_slot[k][s_lblk[q]] = (unsigned char)q;
  __syncthreads();
  // ---- stage 2: output-centric accumulation; item = block pair (lo <= hi) or a block's right-hand side ----
  const int grp = threadIdx.x / 36, el = threadIdx.x % 36;
  const int npairs = L * (L + 1) / 2;
  if (grp < 7) {
    const int i = el / 6, j = el % 6;
    for (int item = grp; item < npairs + L; item += 7) {
      if (item >= npairs) {  // right-hand side of local block l
        if (el >= 6) continue;
        const int l = item - npairs;
        double acc = 0.0;
        for (int k = 0; k < P; ++k) {
          const unsigned char sa = s_slot[k][l];
          if (sa != 255) acc += ent[(size_t)sa * kEntryDoubles + 36 + el];
        }
        if (acc != 0.0) atomicAdd(&d.rhs[s_col[l] + el], acc);
        continue;
      }
      int hi = (int)((sqrt(8.0 * item + 1.0) - 1.0) * 0.5);
      while ((hi + 1) * (hi + 2) / 2 <= item) ++hi;
      while (hi * (hi + 1) / 2 > item) --hi;
      const int lo = item - hi * (hi + 1) / 2;  // lo <= hi, columns ascending: the block sits in S's upper triangle
      const int col_hi = s_col[hi];
      double acc = 0.0;
      for (int k = 0; k < P; ++k) {
        const unsigned char sa = s_slot[k][lo], sb = s_slot[k][hi];
        if (sa == 255 || sb == 255) continue;
        const double* ea = ent + (size_t)sa * kEntryDoubles;
        const double* eb = ent + (size_t)sb * kEntryDoubles;
        acc -= ea[18 + 3 * i] * eb[3 * j] + ea[18 + 3 * i + 1] * eb[3 * j + 1] + ea[18 + 3 * i + 2] * eb[3 * j + 2];
        const int ga = s_ggidx[sa];
        if (lo == hi) {
          if (ga >= 0) acc += gg[(size_t)ga * 36 + el];                                   // group: sum Jg^T Jg
          else acc += ea[42 + i] * ea[42 + j] + ea[48 + i] * ea[48 + j];                   // camera: Jc^T Jc
        } else if (ga < 0 && -2 - ga == col_hi) {                                          // camera x its own group: Jc^T Jg
          acc += ea[42 + i] * ea[54 + j] + ea[48 + i] * ea[60 + j];
        }
      }
      if (acc != 0.0) atomicAdd(&d.S[(size_t)(s_col[lo] + i) * d.nB + col_hi + j], acc);
    }
  }
}

// mirror the upper-triangular block form into the lower triangle, add D^2 on the diagonal, rhs -= g
__global__ void k_ba_finish_S(Dev d, double inv_radius) {
  const uint32_t i = blockIdx.y * blockDim.y + threadIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.nB || j >= d.nB) return;
  if (i > j) d.S[(size_t)i * d.nB + j] = d.S[(size_t)j * d.nB + i];
  if (i == j) {
    d.S[(size_t)i * d.nB + i] += fmin(fmax(d.diag[i], 1e-6), 1e32) * inv_radius;
    d.rhs[i] -= d.g[i];
  }
}

// ---- dense Cholesky + both triangular solves: ONE persistent cooperative kernel -------------------
// A is (n+1) x n row-major: the reduced camera system S with its right-hand side as row n (the same
// contiguous S|rhs block the all-reduce sums).  Right-looking blocked factorisation, NB = 32:
//   per panel k   potrf   every CTA factors the 32x32 diagonal block redundantly in shared memory and
//                         forms its inverse M = L_kk^-1 in the same 32-step loop (one rsqrt per step)
//                 trsm    row tile i (one per CTA): L_ik = A_ik M^T (32^3 MACs) -> Lm      | grid.sync
//                 syrk    trailing tiles (i >= j), four per CTA at a time (256 threads each, 2x2
//                         outputs per thread: one shared-memory operand read per DFMA instead of
//                         three): A_ij -= L_ik L_jk^T                                        | grid.sync
//                 L goes to a SEPARATE matrix Lm, the trailing matrix stays in A.
//   rhs row       carrying b as row n makes the forward substitution L y = b part of the panel updates.
//   backward      L^T x = y by CTA 0, right-looking with the stored inverses of the diagonal blocks.
// One launch instead of 3 per panel + a single-thread triangular solve.
constexpr int NB = 32;
constexpr int kCholGroups = 4;  // syrk tiles in flight per CTA
constexpr size_t kCholSmemBytes = (size_t)(2 + 2 * kCholGroups) * NB * (NB + 1) * sizeof(double) + NB * sizeof(double);
__global__ void __launch_bounds__(1024, 1) k_chol_fused(double* A, double* Lm, double* Linv, int n, double* flag,
                                                        double* x_out) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) double chol_smem[];
  typedef double Tile[NB][NB + 1];
  Tile& T = *(Tile*)(chol_smem);
  Tile& M = *(Tile*)(chol_smem + NB * (NB + 1));
  Tile* G = (Tile*)(chol_smem + 2 * NB * (NB + 1));  // G[2g], G[2g+1]: operand tiles of group g
  double* xk = chol_smem + (size_t)(2 + 2 * kCholGroups) * NB * (NB + 1);
  const int r = threadIdx.y, c = threadIdx.x;
  const int tid = r * NB + c;
  const int nblk = (n + NB - 1) / NB;
  for (int kbi = 0; kbi < nblk; ++kbi) {
    const int k0 = kbi * NB, kb = min(NB, n - k0);
    // ---- potrf: L_kk and M = L_kk^-1 (rows/cols >= kb are identity padding) ----
    T[r][c] = (r < kb && c < kb) ? A[(size_t)(k0 + r) * n + k0 + c] : (r == c ? 1.0 : 0.0);
    M[r][c] = (r == c) ? 1.0 : 0.0;
    __syncthreads();
    for (int j = 0; j < kb; ++j) {
      const double piv = T[j][j];
      const bool bad = !(piv > 0.0);
      const double rs = bad ? 1.0 : rsqrt(piv);
      const double lrj = T[r][j] * rs, lcj = T[c][j] * rs, mjc = M[j][c] * rs;
      const double trc = T[r][c], mrc = M[r][c];
      __syncthreads();
      if (bad && tid == 0 && blockIdx.x == 0) *flag = 1.0;
      if (r == j) {
        M[j][c] = mjc;
        if (c == j) T[j][j] = bad ? 1.0 : piv * rs;
      } else if (r > j) {
        M[r][c] = mrc - lrj * mjc;
        if (c == j) T[r][j] = lrj;
        else if (c > j && c <= r) T[r][c] = trc - lrj * lcj;
      }
      __syncthreads();
    }
    if (blockIdx.x == 0) {
      if (r < kb && c <= r && c < kb) Lm[(size_t)(k0 + r) * n + k0 + c] = T[r][c];
      Linv[(size_t)kbi * NB * NB + r * NB + c] = (c <= r) ? M[r][c] : 0.0;
    }
    // ---- trsm: rows r0 .. n (n = the rhs row), one 32-row tile per CTA ----
    const int r0 = k0 + kb;
    const int tiles_i = (n + 1 - r0 + NB - 1) / NB;
    for (int ti = blockIdx.x; ti < tiles_i; ti += gridDim.x) {
      const int ri = r0 + ti * NB + r;
      __syncthreads();
      G[0][r][c] = (ri <= n && c < kb) ? A[(size_t)ri * n + k0 + c] : 0.0;
      __syncthreads();
      double x = 0.0;
      for (int tt = 0; tt < NB; ++tt) x += G[0][r][tt] * M[c][tt];  // X = A_panel * M^T
      if (ri <= n && c < kb) Lm[(size_t)ri * n + k0 + c] = x;      // L_ik (row n: y_k)
    }
    grid.sync();
    // ---- syrk: A_ij -= L_ik L_jk^T over the trailing tiles; group g = 256 threads works on its own tile ----
    {
      const int g = tid >> 8, gt = tid & 255;
      const int tr = gt >> 4, tc = gt & 15;
      Tile& Xi = G[2 * g];
      Tile& Xj = G[2 * g + 1];
      const int ntiles = tiles_i * (tiles_i + 1) / 2;
      const int stride = gridDim.x * kCholGroups;
      for (int t0 = blockIdx.x * kCholGroups; t0 < ntiles; t0 += stride) {
        const int t = t0 + g;
        int ti = 0, tj = 0;
        if (t < ntiles) {
          ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
          while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
          while (ti * (ti + 1) / 2 > t) --ti;
          tj = t - ti * (ti + 1) / 2;
        }
        __syncthreads();  // the previous round's readers are done
        if (t < ntiles) {
          for (int e = gt; e < NB * NB; e += 256) {
            const int rr = e >> 5, cc = e & 31;
            const int ri = r0 + ti * NB + rr, rj = r0 + tj * NB + rr;
            Xi[rr][cc] = (ri <= n && cc < kb) ? Lm[(size_t)ri * n + k0 + cc] : 0.0;
            Xj[rr][cc] = (rj <= n && cc < kb) ? Lm[(size_t)rj * n + k0 + cc] : 0.0;
          }
        }
        __syncthreads();
        if (t < ntiles) {
          double s00 = 0.0, s01 = 0.0, s10 = 0.0, s11 = 0.0;
          for (int tt = 0; tt < NB; ++tt) {
            const double a0 = Xi[tr][tt], a1 = Xi[tr + 16][tt], b0 = Xj[tc][tt], b1 = Xj[tc + 16][tt];
            s00 += a0 * b0; s01 += a0 * b1; s10 += a1 * b0; s11 += a1 * b1;
          }
          const int row0 = r0 + ti * NB + tr, col0 = r0 + tj * NB + tc;
          if (row0 <= n && col0 < n && col0 <= row0) A[(size_t)row0 * n + col0] -= s00;
          if (row0 <= n && col0 + 16 < n && col0 + 16 <= row0) A[(size_t)row0 * n + col0 + 16] -= s01;
          if (row0 + 16 <= n && col0 < n && col0 <= row0 + 16) A[(size_t)(row0 + 16) * n + col0] -= s10;
          if (row0 + 16 <= n && col0 + 16 < n && col0 + 16 <= row0 + 16) A[(size_t)(row0 + 16) * n + col0 + 16] -= s11;
        }
      }
    }
    grid.sync();
  }
  if (blockIdx.x != 0) return;
  // ---- backward substitution L^T x = y (y = row n of Lm) ----
  for (int j = tid; j < n; j += NB * NB) x_out[j] = Lm[(size_t)n * n + j];
  __syncthreads();
  for (int kbi = nblk - 1; kbi >= 0; --kbi) {
    const int k0 = kbi * NB, kb = min(NB, n - k0);
    M[r][c] = Linv[(size_t)kbi * NB * NB + r * NB + c];
    __syncthreads();
    if (r == 0) {  // x_k = M^T y_k
      double sacc = 0.0;
      for (int tt = 0; tt < kb; ++tt) sacc += M[tt][c] * x_out[k0 + tt];
      xk[c] = (c < kb) ? sacc : 0.0;
    }
    __syncthreads();
    if (r == 0 && c < kb) x_out[k0 + c] = xk[c];
    for (int j = tid; j < k0; j += NB * NB) {  // y_j -= L_kj^T x_k
      double sacc = 0.0;
      for (int tt = 0; tt < kb; ++tt) sacc += Lm[(size_t)(k0 + tt) * n + j] * xk[tt];
      x_out[j] -= sacc;
    }
    __syncthreads();
  }
}

// ---- envelope (skyline) Cholesky: one thread-block CLUSTER, for reduced systems with sparse co-visibility ---------
// Ceres solves the reduced camera system with a sparse Cholesky (SPARSE_SCHUR); the counterpart here keeps the dense
// (n+1) x n storage but only touches the ENVELOPE: row i of S (and of L: the factorisation fills nothing outside it) is
// zero left of first_col(i) = the first camera that shares a point with camera i; intrinsics rows and the right-hand
// side row reach column 0.  At tile granularity: ft[ti] = first column tile of row tile ti, and panel k only involves
// the ACTIVE row tiles R_k = { ti > k : ft[ti] <= k } -- for an image sequence a handful (the band, the intrinsics /
// rhs border, a wrap-around if the sequence closes) instead of all nblk - k.  With so little work per panel the two
// grid-wide barriers of k_chol_fused are what costs; here a panel is
//   potrf   warp 0, the 32 x 32 diagonal tile in registers (lane = row, columns exchanged with shuffles); the rhs row
//           rides along as an extra row when it lies inside the diagonal tile (last panel)
//   trsm    one warp per active row tile: X L_kk^T = A_panel by substitution (lane = row, L_kk broadcast from shared
//           memory); X goes to Lm and, transposed, to shared memory
//   syrk    one warp per pair of active tiles, 4 x 8 outputs per lane: A_ij -= X_i X_j^T
// Every CTA of the cluster repeats potrf and trsm for itself (cheap, and it removes two of the three exchanges); only
// the syrk pairs -- the bulk of the flops -- are dealt round-robin over the cluster's warps, so ONE hardware cluster
// barrier per panel orders "trailing tiles updated" before "next panel loaded".  Data written by another CTA is read
// with ld.global.cg (L2): the SMs' L1 caches are not coherent.  The backward substitution (CTA 0) skips what lies
// outside the envelope too.  The host picks this kernel when every |R_k| <= kEnvMaxActive and the tile-pair count says
// it is cheaper than the dense cooperative kernel.
// Preconditions (envelope_cholesky checks them on the host): n is EVEN -- rows are loaded as double2, so row r starts
// 16-byte aligned only when r * n is even (BA's nB = 6 (C + G) always is); A and Lm hold 64 doubles of slack past
// (n+1) x n (the rhs row is read as whole 32-wide rows); 0 <= ft[t] <= t for the ceil((n+1) / 32) row tiles.  Only
// the lower triangle of A is read.
constexpr int kEnvThreads = 512;
constexpr int kEnvWarps = kEnvThreads / 32;
constexpr int kEnvMaxActive = 24;
constexpr int kEnvMaxCluster = 8;
constexpr size_t kEnvSmemBytes = ((size_t)NB * (NB + 1) + NB + (size_t)kEnvMaxActive * NB * NB) * sizeof(double) + 64 * sizeof(int);
__device__ __forceinline__ void env_cluster_sync(bool clustered) {
  if (clustered) {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  } else {
    __syncthreads();
  }
}
__global__ void __launch_bounds__(kEnvThreads, 1) k_chol_envelope(double* A, double* Lm, int n, const int* __restrict__ ft, double* flag,
                                                                  double* x_out) {
  extern __shared__ __align__(16) double env_smem[];
  typedef double Tile[NB][NB + 1];
  Tile& Ls = *(Tile*)(env_smem);                        // L_kk, row-major (padded)
  double* invd = env_smem + NB * (NB + 1);              // 1 / L_kk[j][j]
  double* Xt = invd + NB;                               // [slot][t][row]: the panel's L_ik, transposed
  int* act = reinterpret_cast<int*>(Xt + (size_t)kEnvMaxActive * NB * NB);  // act[0] = count, act[1..] = tiles
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ncta = gridDim.x, cta = blockIdx.x;         // the grid is one cluster
  const bool clustered = ncta > 1;
  const int nblk = (n + NB - 1) / NB;
  const int ntr = (n + 1 + NB - 1) / NB;                // row tiles including the rhs row n
  for (int kbi = 0; kbi < nblk; ++kbi) {
    const int k0 = kbi * NB, kb = min(NB, n - k0);
    if (warp == 1) {  // the panel's active row tiles, ascending
      int cnt = 0;
      for (int base = 0; base < ntr; base += 32) {
        const int ti = base + lane;
        const bool a = ti > kbi && ti < ntr && ft[ti] <= kbi;
        const unsigned m = __ballot_sync(0xffffffffu, a);
        if (a) act[1 + cnt + __popc(m & ((1u << lane) - 1u))] = ti;
        cnt += __popc(m);
      }
      if (lane == 0) act[0] = cnt;
    }
    if (warp == 0) {  // ---- potrf of the diagonal tile; lane kb carries the rhs row when it lies in this tile ----
      // lane = row, the row in registers; column j reaches the other lanes through shared memory (one broadcast read
      // per update).  Every lane updates all 32 entries of its row: what lands above the diagonal or in the padding
      // is never read, and leaving the predicates out keeps the unrolled code small (it runs once per panel, from
      // the instruction cache's point of view always cold).
      const bool rhs_lane = kb < NB && lane == kb && k0 + kb == n;
      const bool real = lane < kb || rhs_lane;
      double a[NB];
      {
        const double2* src = reinterpret_cast<const double2*>(A + (size_t)(k0 + (real ? lane : 0)) * n + k0);
#pragma unroll
        for (int c = 0; c < NB; c += 2) {
          const double2 v = __ldcg(src + c / 2);
          a[c] = (real && c < kb) ? v.x : (lane == c ? 1.0 : 0.0);
          a[c + 1] = (real && c + 1 < kb) ? v.y : (lane == c + 1 ? 1.0 : 0.0);
        }
      }
      double* colb = Xt;  // 2 x 32 doubles of scratch (Xt is not in use before the trsm)
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        if (j < kb) {  // (warp-uniform) columns beyond kb are identity padding
          double* cb = colb + (j & 1) * 2 * NB;
          if (lane == j) cb[NB] = a[j];
          __syncwarp();
          const double piv = cb[NB];
          const bool bad = !(piv > 0.0);
          const double rs = bad ? 1.0 : rsqrt(piv);
          if (bad && lane == 0 && cta == 0) *flag = 1.0;
          double lrj = a[j] * rs;                       // L[r][j] for r > j
          if (lane == j) { lrj = bad ? 1.0 : piv * rs; invd[j] = rs; }
          a[j] = lrj;
          cb[lane] = lrj;
          __syncwarp();
#pragma unroll
          for (int c = j + 1; c < NB; ++c) a[c] -= lrj * cb[c];
        } else if (lane == j) {
          invd[j] = 1.0;
        }
      }
#pragma unroll
      for (int c = 0; c < NB; ++c) {
        const double v = lane < kb ? (c <= lane ? a[c] : 0.0) : (c == lane ? 1.0 : 0.0);  // the rhs lane is not a row of L_kk
        Ls[lane][c] = v;
        if (cta == 0 && real && c < kb && c <= lane) Lm[(size_t)(k0 + lane) * n + k0 + c] = a[c];
      }
    }
    __syncthreads();
    const int nact = act[0];
    // ---- trsm: a warp per active tile (every CTA for itself) ----
    for (int slot = warp; slot < nact; slot += kEnvWarps) {
      const int ti = act[1 + slot];
      const int row = ti * NB + lane;
      const bool valid = row <= n;
      double a[NB];
      {
        const double2* src = reinterpret_cast<const double2*>(A + (size_t)(valid ? row : n) * n + k0);
#pragma unroll
        for (int c = 0; c < NB; c += 2) {
          const double2 v = __ldcg(src + c / 2);
          a[c] = (valid && c < kb) ? v.x : 0.0;
          a[c + 1] = (valid && c + 1 < kb) ? v.y : 0.0;
        }
      }
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const double xj = a[j] * invd[j];
        a[j] = xj;
#pragma unroll
        for (int m = j + 1; m < NB; ++m) a[m] -= xj * Ls[m][j];
      }
      double* xt = Xt + (size_t)slot * NB * NB;
#pragma unroll
      for (int c = 0; c < NB; ++c) {
        xt[c * NB + lane] = a[c];
        if (cta == 0 && valid && c < kb) Lm[(size_t)row * n + k0 + c] = a[c];
      }
    }
    __syncthreads();
    // ---- syrk over the pairs (ia >= ib) of active tiles, dealt over the cluster's warps;
    //      lane = (4 rows, 8 columns) of the 32 x 32 target ----
    {
      const int npairs = nact * (nact + 1) / 2;
      const int lr = lane >> 2, lc = lane & 3;
      for (int pi = warp * ncta + cta; pi < npairs; pi += kEnvWarps * ncta) {
        int ia = (int)((sqrtf(8.f * (float)pi + 1.f) - 1.f) * 0.5f);
        while ((ia + 1) * (ia + 2) / 2 <= pi) ++ia;
        while (ia * (ia + 1) / 2 > pi) --ia;
        const int ib = pi - ia * (ia + 1) / 2;
        const double* xa = Xt + (size_t)ia * NB * NB + 4 * lr;
        const double* xb = Xt + (size_t)ib * NB * NB + 8 * lc;
        double acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;
#pragma unroll 4
        for (int t = 0; t < NB; ++t) {
          const double2 a01 = *reinterpret_cast<const double2*>(xa + t * NB);
          const double2 a23 = *reinterpret_cast<const double2*>(xa + t * NB + 2);
          const double av[4] = {a01.x, a01.y, a23.x, a23.y};
          double bv[8];
#pragma unroll
          for (int j = 0; j < 8; j += 2) {
            const double2 b2 = *reinterpret_cast<const double2*>(xb + t * NB + j);
            bv[j] = b2.x; bv[j + 1] = b2.y;
          }
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] += av[i] * bv[j];
        }
        const int row0 = act[1 + ia] * NB + 4 * lr, col0 = act[1 + ib] * NB + 8 * lc;
        // read-modify-write of the target: all loads first (the compiler will not hoist a load over a store that
        // may alias it, and 32 serialised L2 round trips would cost more than the tile product)
        double old[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int row = row0 + i, col = col0 + j;
            old[i][j] = (row <= n && col < n && col <= row) ? __ldcg(&A[(size_t)row * n + col]) : 0.0;
          }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int row = row0 + i, col = col0 + j;
            if (row <= n && col < n && col <= row) A[(size_t)row * n + col] = old[i][j] - acc[i][j];
          }
      }
    }
    env_cluster_sync(clustered);
  }
  if (cta != 0) return;
  // ---- backward substitution L^T x = y (y = row n of Lm), inside the envelope ----
  for (int j = tid; j < n; j += kEnvThreads) x_out[j] = __ldcg(&Lm[(size_t)n * n + j]);
  __syncthreads();
  for (int kbi = nblk - 1; kbi >= 0; --kbi) {
    const int k0 = kbi * NB, kb = min(NB, n - k0);
    if (warp == 0) {  // x_k = L_kk^-T y_k: lane c holds column c of L_kk (col[j] = L[j][c], zero above the diagonal)
      double col[NB];
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const double v = __ldcg(&Lm[(size_t)(k0 + min(j, kb - 1)) * n + k0 + min(lane, kb - 1)]);
        col[j] = (j < kb && lane < kb && lane <= j) ? v : (j == lane ? 1.0 : 0.0);
      }
      double y = lane < kb ? __ldcg(&x_out[k0 + lane]) : 0.0;
      double diag = 1.0;
#pragma unroll
      for (int j = 0; j < NB; ++j) diag = (j == lane) ? col[j] : diag;
      const double inv = 1.0 / diag;
      double* xb = Xt;  // scratch: x_k as it is solved, last entry first
#pragma unroll
      for (int j = NB - 1; j >= 0; --j) {
        if (lane == j) xb[j] = y * inv;
        __syncwarp();
        y -= col[j] * xb[j];   // lanes > j: col[j] = 0; lane j: y becomes 0 and is not used again
      }
      __syncwarp();
      const double x = xb[lane];
      if (lane < kb) x_out[k0 + lane] = x;
      invd[lane] = lane < kb ? x : 0.0;  // x_k for the update below
    }
    __syncthreads();
    const int lo = min(ft[kbi] * NB, k0);
    for (int j = lo + tid; j < k0; j += kEnvThreads) {  // y_j -= L_kj^T x_k (loads batched: they are L2 round trips)
      double lv[NB];
#pragma unroll
      for (int tt = 0; tt < NB; ++tt) lv[tt] = tt < kb ? __ldcg(&Lm[(size_t)(k0 + tt) * n + j]) : 0.0;
      double sacc = 0.0;
#pragma unroll
      for (int tt = 0; tt < NB; ++tt) sacc += lv[tt] * invd[tt];
      x_out[j] = __ldcg(&x_out[j]) - sacc;
    }
    __syncthreads();
  }
}

// ---- back substitution ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_ba_backsub(Dev d, double inv_radius) {
  const uint32_t ip = blockIdx.x * blockDim.x + threadIdx.x;
  if (ip >= d.n_pts) return;
  const size_t pcol = (size_t)d.nB + 3 * (size_t)ip;
  const uint32_t b = d.pt_ofs[ip], e = d.pt_ofs[ip + 1];
  if (b == e) {  // no observation, so no Schur kernel visits the point: V = D^2 (its g_p is 0, so is its step)
    for (int i = 0; i < 9; ++i) d.Vinv[9 * (size_t)ip + i] = (i % 4) ? 0.0 : 1.0 / (fmin(fmax(d.diag[pcol + i / 4], 1e-6), 1e32) * inv_radius);
  }
  double t3[3] = {-d.g[pcol], -d.g[pcol + 1], -d.g[pcol + 2]};
  for (uint32_t t = b; t < e; ++t) {
    double Jc[12], Jg[12], Jp[6], r[2];
    uint32_t cc;
    int cg;
    scaled_jacobian(d, d.pt_obs[t], Jc, Jg, Jp, r, &cc, &cg);
    double m[2] = {0, 0};
    for (int a = 0; a < 2; ++a) {
      for (int k = 0; k < 6; ++k) m[a] += Jc[6 * a + k] * d.delta[cc + k];
      if (cg >= 0)
        for (int k = 0; k < 6; ++k) m[a] += Jg[6 * a + k] * d.delta[cg + k];
    }
    for (int k = 0; k < 3; ++k) t3[k] -= Jp[k] * m[0] + Jp[3 + k] * m[1];
  }
  const double* Vi = d.Vinv + 9 * (size_t)ip;
  for (int i = 0; i < 3; ++i) d.delta[pcol + i] = Vi[3 * i] * t3[0] + Vi[3 * i + 1] * t3[1] + Vi[3 * i + 2] * t3[2];
}

// ---- pose-centre priors (ViewPriors / GPS): a camera-only residual block per prior ------------------------
// mode 0: cost at (poses) -> out[0] ; mode 1: gradient + diag(J^T J), unscaled -> gu, du ; mode 2: U block of S (scaled)
__global__ void k_ba_priors(Dev d, const double* poses, int mode, double* out_cost) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= d.n_priors) return;
  const uint32_t cam = d.prior_cam[k];
  double r[3], J[18];
  prior_residual_jacobian(poses + 6 * (size_t)cam, d.prior_center + 3 * (size_t)k, d.prior_weight + 3 * (size_t)k, r, mode ? J : nullptr);
  double rho1;
  const double rho = huber_rho(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], d.prior_huber_a, &rho1);
  if (mode == 0) {
    atomicAdd(out_cost, 0.5 * rho);
  } else if (mode == 1) {
    for (int q = 0; q < 6; ++q) {
      atomicAdd(&d.gu[6 * (size_t)cam + q], rho1 * (J[q] * r[0] + J[6 + q] * r[1] + J[12 + q] * r[2]));
      atomicAdd(&d.du[6 * (size_t)cam + q], rho1 * (J[q] * J[q] + J[6 + q] * J[6 + q] + J[12 + q] * J[12 + q]));
    }
  } else {
    const double* sc = d.scale + 6 * (size_t)cam;
    double blk[36];
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j)
        blk[6 * i + j] = rho1 * sc[i] * sc[j] * (J[i] * J[j] + J[6 + i] * J[6 + j] + J[12 + i] * J[12 + j]);
    add_block_upper(d.S, d.nB, 6 * cam, 6 * cam, blk, 1.0);
  }
}

// ---- candidate parameters, step norms, model cost change ---------------------------------------------
__global__ void __launch_bounds__(256) k_ba_update(Dev d, double inv_radius) {
  __shared__ double sm[8];
  const size_t nparam = (size_t)d.nB + 3 * (size_t)d.n_pts;
  double mcc = 0, dn = 0, xn = 0;
  for (size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x; j < nparam; j += (size_t)gridDim.x * blockDim.x) {
    const double D2 = fmin(fmax(d.diag[j], 1e-6), 1e32) * inv_radius;
    const double dl = d.delta[j];
    const double dx = dl * d.scale[j];
    const bool counted = d.owns_shared || j >= d.nB;
    if (counted) mcc += dl * (D2 * dl - d.g[j]);
    double x;
    if (j < 6 * (size_t)d.n_cams) { x = d.poses[j]; d.poses_new[j] = x + dx; }
    else if (j < d.nB) { x = d.intr[j - 6 * (size_t)d.n_cams]; d.intr_new[j - 6 * (size_t)d.n_cams] = x + dx; }
    else { x = d.pts[j - d.nB]; d.pts_new[j - d.nB] = x + dx; }
    if (counted) {
      dn += dx * dx;
      xn += x * x;
    }
  }
  mcc = block_sum(mcc, sm);
  dn = block_sum(dn, sm);
  xn = block_sum(xn, sm);
  if (threadIdx.x == 0) {
    atomicAdd(&d.scal[1], mcc);
    atomicAdd(&d.scal[2], dn);
    atomicAdd(&d.scal[3], xn);
  }
}

}  // namespace ba

int dense_cholesky_grid(r3d_ctx* ctx, DeviceWorker& w, int* grid) {
  int per_sm = 0;
  R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(ba::k_chol_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba::kCholSmemBytes));
  R3D_CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ba::k_chol_fused, 1024, ba::kCholSmemBytes));
  if (per_sm < 1) return fail(ctx, R3D_ERR_CUDA, "dense Cholesky: k_chol_fused does not fit on an SM");
  if (*grid == 0) *grid = w.sm_count;
  if (*grid < 1 || *grid > per_sm * w.sm_count)
    return fail(ctx, R3D_ERR_INVALID, "dense Cholesky: " + std::to_string(*grid) + " CTAs cannot be co-resident");
  return R3D_OK;
}

int dense_cholesky(r3d_ctx* ctx, DeviceWorker& w, double* A, double* L, double* Linv, int n, double* flag, double* x, int grid) {
  static_assert(kCholNB == ba::NB, "Linv layout");
  int rc;
  if ((rc = dense_cholesky_grid(ctx, w, &grid))) return rc;
  void* args[] = {&A, &L, &Linv, &n, &flag, &x};
  R3D_CUDA_TRY(ctx, cudaLaunchCooperativeKernel((void*)ba::k_chol_fused, dim3(grid), dim3(32, 32), args, ba::kCholSmemBytes,
                                                w.stream));
  return R3D_OK;
}

int envelope_cholesky(r3d_ctx* ctx, DeviceWorker& w, double* A, double* L, int n, const int* ft, int ctas, double* flag, double* x) {
  if (ctas < 1 || ctas > ba::kEnvMaxCluster)
    return fail(ctx, R3D_ERR_INVALID, "envelope Cholesky: cluster of " + std::to_string(ctas) + " CTAs");
  if (n % 2) return fail(ctx, R3D_ERR_INVALID, "envelope Cholesky: n must be even");
  R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(ba::k_chol_envelope, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba::kEnvSmemBytes));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(ctas);
  cfg.blockDim = dim3(ba::kEnvThreads);
  cfg.dynamicSmemBytes = ba::kEnvSmemBytes;
  cfg.stream = w.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = ctas;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  R3D_CUDA_TRY(ctx, cudaLaunchKernelEx(&cfg, ba::k_chol_envelope, A, L, n, ft, flag, x));
  return R3D_OK;
}

}  // namespace r3d

// ------------------------------------------------------------------------------------------------
using namespace r3d;
using r3d::ba::Dev;

namespace {

struct DeviceArrays {  // blocks come from (and return to) the worker's size-bucketed pool: no cudaMalloc per call
  DeviceWorker* w = nullptr;
  std::vector<void*> ptrs;
  ~DeviceArrays() {
    if (!w) return;
    cudaStreamSynchronize(w->stream);
    for (void* p : ptrs) pool_release(*w, p);
  }
  template <typename T>
  cudaError_t alloc(T** p, size_t n) {
    *p = (T*)pool_alloc(*w, std::max<size_t>(n, 1) * sizeof(T));
    if (!*p) return cudaErrorMemoryAllocation;
    ptrs.push_back(*p);
    return cudaSuccess;
  }
};

struct BatchPlan {  // device tables of the batched Schur kernel + the points that go through the general CTA kernel
  std::vector<uint32_t> first_cam;  // per camera: the lowest-numbered camera it shares a point with (envelope of S)
  r3d::ba::BatchTables t{};
  uint32_t n_batches = 0;
  const uint32_t* d_long = nullptr;  // point ids for k_ba_schur_cta
  uint32_t n_long = 0, long_cap = 1; // their number and longest track
  bool want_batched = true;          // false: every point takes the CTA kernel (R3D_BA_SCHUR=point)
};

int setup_problem(r3d_ctx* ctx, DeviceWorker& w, const r3d_ba_problem* p, DeviceArrays& mem, Dev& d, bool refine_intr,
                  double huber_a, bool full, uint32_t* max_obs_out = nullptr, BatchPlan* plan = nullptr) {
  if (!p || !p->poses || !p->intrinsics || !p->points || !p->obs_cam || !p->obs_pt || !p->cam_intr || !p->obs_xy)
    return fail(ctx, R3D_ERR_INVALID, "bundle adjustment: NULL array in the problem");
  for (uint64_t o = 0; o < p->n_obs; ++o)
    if (p->obs_cam[o] >= p->n_cams || p->obs_pt[o] >= p->n_pts) return fail(ctx, R3D_ERR_INVALID, "bundle adjustment: observation index out of range");
  for (uint32_t c = 0; c < p->n_cams; ++c)
    if (p->cam_intr[c] >= p->n_intr) return fail(ctx, R3D_ERR_INVALID, "bundle adjustment: intrinsic group out of range");
  std::memset(&d, 0, sizeof(d));
  d.n_cams = p->n_cams; d.n_pts = p->n_pts; d.n_intr = p->n_intr; d.n_obs = p->n_obs;
  d.refine_intr = refine_intr ? 1u : 0u;
  d.nB = 6 * p->n_cams + (refine_intr ? 6 * p->n_intr : 0);
  d.huber_a = huber_a;
  d.prior_huber_a = 0.0;
  d.owns_shared = ctx->comm_rank == 0 ? 1u : 0u;
  const size_t nparam = (size_t)d.nB + 3 * (size_t)p->n_pts;
  uint32_t *oc, *op, *ci, *pofs, *pobs;
  double2* oxy;
  R3D_CUDA_TRY(ctx, mem.alloc(&d.poses, 6 * (size_t)p->n_cams));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.intr, 6 * (size_t)p->n_intr));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.pts, 3 * (size_t)p->n_pts));
  R3D_CUDA_TRY(ctx, mem.alloc(&oc, p->n_obs));
  R3D_CUDA_TRY(ctx, mem.alloc(&op, p->n_obs));
  R3D_CUDA_TRY(ctx, mem.alloc(&ci, p->n_cams));
  R3D_CUDA_TRY(ctx, mem.alloc(&oxy, p->n_obs));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.scal, 8));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d.poses, p->poses, 6 * (size_t)p->n_cams * 8, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d.intr, p->intrinsics, 6 * (size_t)p->n_intr * 8, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d.pts, p->points, 3 * (size_t)p->n_pts * 8, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(oc, p->obs_cam, p->n_obs * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(op, p->obs_pt, p->n_obs * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(ci, p->cam_intr, (size_t)p->n_cams * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(oxy, p->obs_xy, p->n_obs * 16, cudaMemcpyHostToDevice, w.stream));
  d.obs_cam = oc; d.obs_pt = op; d.cam_intr = ci; d.obs_xy = oxy;
  if (p->intr_model) {
    for (uint32_t g = 0; g < p->n_intr; ++g)
      if (p->intr_model[g] < 1 || p->intr_model[g] > 5) return fail(ctx, R3D_ERR_INVALID, "bundle adjustment: unknown camera model");
    uint8_t* dm;
    R3D_CUDA_TRY(ctx, mem.alloc(&dm, p->n_intr));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(dm, p->intr_model, p->n_intr, cudaMemcpyHostToDevice, w.stream));
    d.intr_model = dm;
  }
  if (p->intrinsics_ext) {
    double* de;
    R3D_CUDA_TRY(ctx, mem.alloc(&de, 2 * (size_t)p->n_intr));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(de, p->intrinsics_ext, 2 * (size_t)p->n_intr * 8, cudaMemcpyHostToDevice, w.stream));
    d.intr_ext = de;
  }
  if (p->n_priors) {
    if (!p->prior_cam || !p->prior_center || !p->prior_weight) return fail(ctx, R3D_ERR_INVALID, "bundle adjustment: NULL prior array");
    for (uint32_t k = 0; k < p->n_priors; ++k)
      if (p->prior_cam[k] >= p->n_cams) return fail(ctx, R3D_ERR_INVALID, "bundle adjustment: prior camera out of range");
    uint32_t* pc;
    double *pce, *pw;
    R3D_CUDA_TRY(ctx, mem.alloc(&pc, p->n_priors));
    R3D_CUDA_TRY(ctx, mem.alloc(&pce, 3 * (size_t)p->n_priors));
    R3D_CUDA_TRY(ctx, mem.alloc(&pw, 3 * (size_t)p->n_priors));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(pc, p->prior_cam, (size_t)p->n_priors * 4, cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(pce, p->prior_center, 3 * (size_t)p->n_priors * 8, cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(pw, p->prior_weight, 3 * (size_t)p->n_priors * 8, cudaMemcpyHostToDevice, w.stream));
    d.n_priors = p->n_priors; d.prior_cam = pc; d.prior_center = pce; d.prior_weight = pw;
  }
  if (!full) return R3D_OK;
  if (p->n_obs > 0xfffffff0ull) return fail(ctx, R3D_ERR_UNSUPPORTED, "bundle adjustment: more than 2^32 observations");
  // point -> observation CSR (host counting sort)
  std::vector<uint32_t> hofs((size_t)p->n_pts + 1, 0), hobs(p->n_obs);
  for (uint64_t o = 0; o < p->n_obs; ++o) hofs[p->obs_pt[o] + 1]++;
  uint32_t maxobs = 0;
  for (uint32_t i = 0; i < p->n_pts; ++i) { maxobs = std::max(maxobs, hofs[i + 1]); hofs[i + 1] += hofs[i]; }
  if (max_obs_out) *max_obs_out = maxobs;
  {
    std::vector<uint32_t> pos(hofs.begin(), hofs.end() - 1);
    for (uint64_t o = 0; o < p->n_obs; ++o) hobs[pos[p->obs_pt[o]]++] = (uint32_t)o;
  }
  R3D_CUDA_TRY(ctx, mem.alloc(&pofs, hofs.size()));
  R3D_CUDA_TRY(ctx, mem.alloc(&pobs, hobs.size()));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(pofs, hofs.data(), hofs.size() * 4, cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(pobs, hobs.data(), hobs.size() * 4, cudaMemcpyHostToDevice, w.stream));
  // ---- plan of the batched Schur kernel (static per problem): camera-sorted processing order, batches that
  //      respect the kernel's shared-memory limits, each batch's sorted block columns, every entry's local block
  std::vector<uint32_t> h_order, h_ent_start;
  std::vector<r3d::ba::BatchDesc> h_batches;
  std::vector<int> h_cols;
  std::vector<unsigned char> h_lblk;
  std::vector<uint32_t> h_long;
  if (plan) {
    using namespace r3d::ba;
    const uint32_t n_pts = p->n_pts;
    const int threads = std::max(1, ctx->host_threads);
    plan->first_cam.resize(p->n_cams);
    for (uint32_t c = 0; c < p->n_cams; ++c) plan->first_cam[c] = c;
    for (uint32_t i = 0; i < n_pts; ++i) {
      uint32_t mn = p->n_cams;
      for (uint32_t t = hofs[i]; t < hofs[i + 1]; ++t) mn = std::min(mn, p->obs_cam[hobs[t]]);
      for (uint32_t t = hofs[i]; t < hofs[i + 1]; ++t) {
        uint32_t& f = plan->first_cam[p->obs_cam[hobs[t]]];
        f = std::min(f, mn);
      }
    }
    // (0) which points the batched kernel can take: <= 32 observations, <= 2 intrinsic groups, no camera twice.
    //     Everything else (long tracks first of all) goes to the general CTA-per-point kernel.
    std::vector<uint32_t> key(n_pts, 0), nent(n_pts, 0);
    std::vector<uint8_t> elig(n_pts, 0);
    const uint32_t kSlab = 4096;
    const size_t n_slabs = ((size_t)n_pts + kSlab - 1) / kSlab;
    parallel_for(threads, n_slabs, [&](size_t sl) {
      const uint32_t i1 = (uint32_t)std::min<size_t>((sl + 1) * kSlab, n_pts);
      for (uint32_t i = (uint32_t)(sl * kSlab); i < i1; ++i) {
        const uint32_t nobs = hofs[i + 1] - hofs[i];
        if (!plan->want_batched || nobs > 32 || nobs == 0) continue;
        uint32_t mn = p->n_cams;
        int g0 = -1, g1 = -1, ng = 0;
        bool ok = true;
        for (uint32_t t = hofs[i]; t < hofs[i + 1] && ok; ++t) {
          const uint32_t cam = p->obs_cam[hobs[t]];
          mn = std::min(mn, cam);
          for (uint32_t u = hofs[i]; u < t; ++u)
            if (p->obs_cam[hobs[u]] == cam) ok = false;  // a camera sees the point twice
          if (refine_intr) {
            const int g = (int)p->cam_intr[cam];
            if (g != g0 && g != g1) {
              if (g0 < 0) g0 = g; else if (g1 < 0) g1 = g; else ok = false;  // > 2 groups
              ++ng;
            }
          }
        }
        if (!ok) continue;
        elig[i] = 1;
        key[i] = mn;
        nent[i] = nobs + (uint32_t)ng;
      }
    });
    // (1) processing order of the eligible points: counting sort by the smallest camera that sees them
    {
      std::vector<uint32_t> bucket((size_t)p->n_cams + 2, 0);
      uint32_t n_el = 0;
      for (uint32_t i = 0; i < n_pts; ++i)
        if (elig[i]) { bucket[key[i] + 1]++; ++n_el; }
      for (size_t c = 0; c + 1 < bucket.size(); ++c) bucket[c + 1] += bucket[c];
      h_order.resize(n_el);
      for (uint32_t i = 0; i < n_pts; ++i)
        if (elig[i]) h_order[bucket[key[i]]++] = i;
    }
    const uint32_t n_el = (uint32_t)h_order.size();
    // (2) batches: consecutive ordered points, cut by the point, entry and distinct-block capacities of the kernel
    //     (a stamp per 6-wide block tells whether the open batch already holds it)
    h_ent_start.assign((size_t)n_el + 1, 0);
    {
      std::vector<uint32_t> stamp((size_t)p->n_cams + p->n_intr, 0xffffffffu);
      BatchDesc cur{0, 0, 0, 0};
      uint32_t ent_run = 0, cur_blocks = 0, batch_id = 0;
      for (uint32_t k = 0; k < n_el; ++k) {
        const uint32_t ip = h_order[k];
        const uint32_t ne = nent[ip];
        auto count_new = [&](bool mark) {
          uint32_t fresh = 0;
          for (uint32_t t = hofs[ip]; t < hofs[ip + 1]; ++t) {
            const uint32_t cam = p->obs_cam[hobs[t]];
            const uint32_t blocks[2] = {cam, p->n_cams + p->cam_intr[cam]};
            for (int q = 0; q < (refine_intr ? 2 : 1); ++q)
              if (stamp[blocks[q]] != batch_id && stamp[blocks[q]] != (batch_id | 0x80000000u)) {
                ++fresh;
                if (mark) stamp[blocks[q]] = batch_id;
                else stamp[blocks[q]] = batch_id | 0x80000000u;  // provisional: counted once within this point
              }
          }
          if (!mark)  // undo the provisional marks
            for (uint32_t t = hofs[ip]; t < hofs[ip + 1]; ++t) {
              const uint32_t cam = p->obs_cam[hobs[t]];
              const uint32_t blocks[2] = {cam, p->n_cams + p->cam_intr[cam]};
              for (int q = 0; q < (refine_intr ? 2 : 1); ++q)
                if (stamp[blocks[q]] == (batch_id | 0x80000000u)) stamp[blocks[q]] = 0xffffffffu;
            }
          return fresh;
        };
        const uint32_t fresh = count_new(false);
        if (cur.count && (cur.count == (uint32_t)kBatchPoints || (ent_run - cur.ent_first) + ne > (uint32_t)kBatchEntries ||
                          cur_blocks + fresh > (uint32_t)kBatchBlocks)) {
          h_batches.push_back(cur);
          cur = BatchDesc{k, 0, ent_run, 0};
          cur_blocks = 0;
          ++batch_id;
        }
        cur_blocks += count_new(true);
        h_ent_start[k] = ent_run;
        ent_run += ne;
        cur.count++;
      }
      h_ent_start[n_el] = ent_run;
      if (cur.count) h_batches.push_back(cur);
      h_lblk.assign(ent_run, 0);
    }
    // (3) per batch, in parallel: sorted distinct block columns and every entry's index into them
    h_cols.assign(h_batches.size() * kBatchBlocks, 0);
    parallel_for(threads, h_batches.size(), [&](size_t bi) {
      BatchDesc& bd = h_batches[bi];
      int cols[kBatchEntries * 2];
      int nc = 0;
      for (uint32_t k = 0; k < bd.count; ++k) {
        const uint32_t ip = h_order[bd.first + k];
        for (uint32_t t = hofs[ip]; t < hofs[ip + 1]; ++t) {
          const uint32_t cam = p->obs_cam[hobs[t]];
          cols[nc++] = (int)(6 * cam);
          if (refine_intr) cols[nc++] = (int)(6 * p->n_cams + 6 * p->cam_intr[cam]);
        }
      }
      std::sort(cols, cols + nc);
      nc = (int)(std::unique(cols, cols + nc) - cols);  // <= kBatchBlocks by construction of the batches
      bd.nblk = (uint32_t)nc;
      std::copy(cols, cols + nc, h_cols.begin() + bi * kBatchBlocks);
      unsigned char* lb = h_lblk.data() + bd.ent_first;
      for (uint32_t k = 0; k < bd.count; ++k) {
        const uint32_t ip = h_order[bd.first + k];
        int g0 = -1, g1 = -1;
        for (uint32_t t = hofs[ip]; t < hofs[ip + 1]; ++t) {
          const uint32_t cam = p->obs_cam[hobs[t]];
          *lb++ = (unsigned char)(std::lower_bound(cols, cols + nc, (int)(6 * cam)) - cols);
          if (refine_intr) {
            const int gc = (int)(6 * p->n_cams + 6 * p->cam_intr[cam]);
            if (gc != g0 && gc != g1) { if (g0 < 0) g0 = gc; else g1 = gc; }
          }
        }
        for (int gc : {g0, g1})
          if (gc >= 0) *lb++ = (unsigned char)(std::lower_bound(cols, cols + nc, gc) - cols);
      }
    });
    // (4) the rest: listed for the CTA-per-point kernel, longest tracks first
    for (uint32_t i = 0; i < n_pts; ++i)
      if (!elig[i] && hofs[i + 1] > hofs[i]) {
        h_long.push_back(i);
        plan->long_cap = std::max(plan->long_cap, hofs[i + 1] - hofs[i]);
      }
    std::stable_sort(h_long.begin(), h_long.end(), [&](uint32_t a, uint32_t b) { return hofs[a + 1] - hofs[a] > hofs[b + 1] - hofs[b]; });
    if (!h_batches.empty()) {
      uint32_t *d_order, *d_ent_start;
      BatchDesc* d_batches;
      int* d_cols;
      unsigned char* d_lblk;
      R3D_CUDA_TRY(ctx, mem.alloc(&d_order, h_order.size()));
      R3D_CUDA_TRY(ctx, mem.alloc(&d_ent_start, h_ent_start.size()));
      R3D_CUDA_TRY(ctx, mem.alloc(&d_batches, h_batches.size()));
      R3D_CUDA_TRY(ctx, mem.alloc(&d_cols, h_cols.size()));
      R3D_CUDA_TRY(ctx, mem.alloc(&d_lblk, h_lblk.size()));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_order, h_order.data(), h_order.size() * 4, cudaMemcpyHostToDevice, w.stream));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ent_start, h_ent_start.data(), h_ent_start.size() * 4, cudaMemcpyHostToDevice, w.stream));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_batches, h_batches.data(), h_batches.size() * sizeof(BatchDesc), cudaMemcpyHostToDevice, w.stream));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_cols, h_cols.data(), h_cols.size() * sizeof(int), cudaMemcpyHostToDevice, w.stream));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_lblk, h_lblk.data(), h_lblk.size(), cudaMemcpyHostToDevice, w.stream));
      plan->t = BatchTables{d_batches, d_order, d_ent_start, d_cols, d_lblk};
      plan->n_batches = (uint32_t)h_batches.size();
    }
    if (!h_long.empty()) {
      uint32_t* d_long;
      R3D_CUDA_TRY(ctx, mem.alloc(&d_long, h_long.size()));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_long, h_long.data(), h_long.size() * 4, cudaMemcpyHostToDevice, w.stream));
      plan->d_long = d_long;
      plan->n_long = (uint32_t)h_long.size();
    }
  }
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));  // hofs / hobs and the plan vectors are locals
  d.pt_ofs = pofs; d.pt_obs = pobs;
  R3D_CUDA_TRY(ctx, mem.alloc(&d.poses_new, 6 * (size_t)p->n_cams));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.intr_new, 6 * (size_t)p->n_intr));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.pts_new, 3 * (size_t)p->n_pts));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.scale, nparam));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.gu, nparam));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.du, nparam));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.g, nparam));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.diag, nparam));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.delta, nparam));
  R3D_CUDA_TRY(ctx, mem.alloc(&d.S, (size_t)d.nB * d.nB + d.nB + 64));  // S | rhs contiguous: one all-reduce (+ slack: k_chol_envelope reads whole 32-wide rows)
  d.rhs = d.S + (size_t)d.nB * d.nB;
  R3D_CUDA_TRY(ctx, mem.alloc(&d.Vinv, 9 * (size_t)p->n_pts));
  // intrinsics that are not refined never enter the parameter vector: the candidate copy is constant
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d.intr_new, d.intr, 6 * (size_t)p->n_intr * 8, cudaMemcpyDeviceToDevice, w.stream));
  return R3D_OK;
}

enum CholChoice { kCholDense, kCholEnvelope, kCholAuto };

struct StepPlan {  // what one LM step needs beyond Dev: the Schur plan, the CTA kernel's scratch, the Cholesky's
  BatchPlan plan;
  uint32_t long_grid = 0;
  double* long_scr = nullptr;
  int* long_cols = nullptr;
  double *Lm = nullptr, *Linv = nullptr;
  bool use_env = false;
  int env_ctas = r3d::ba::kEnvMaxCluster;  // CTAs of the envelope kernel's cluster
  int* ft = nullptr;
};

// after setup_problem(..., &s.plan): scratch of both Schur kernels and of the linear solve; the Cholesky kernel
// (envelope only where its active-tile limit holds)
int setup_step(r3d_ctx* ctx, DeviceWorker& w, const r3d_ba_problem* p, DeviceArrays& mem, const Dev& d, CholChoice chol,
               StepPlan& s) {
  int rc;
  const BatchPlan& plan = s.plan;
  if (plan.n_batches)
    R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(r3d::ba::k_ba_schur_batched, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)r3d::ba::kBatchSmemBytes));
  // scratch of the CTA-per-point kernel: one slice of `long_cap` observations per CTA of its (persistent) grid
  if (plan.n_long) {
    s.long_grid = std::min<uint32_t>(plan.n_long, (uint32_t)w.sm_count * 8u);
    const size_t per_cta = (size_t)plan.long_cap * (r3d::ba::kObsDoubles + 36);
    // keep the scratch within ~1 GB whatever the track length
    while (s.long_grid > 1 && per_cta * s.long_grid * sizeof(double) > ((size_t)1 << 30)) s.long_grid /= 2;
    R3D_CUDA_TRY(ctx, mem.alloc(&s.long_scr, per_cta * s.long_grid));
    R3D_CUDA_TRY(ctx, mem.alloc(&s.long_cols, (size_t)plan.long_cap * 3 * s.long_grid));
  }
  const int nB = (int)d.nB;
  // Cholesky scratch: L (with the forward-substituted rhs as row nB) and the inverses of its diagonal blocks
  const int chol_blocks = (nB + r3d::ba::NB - 1) / r3d::ba::NB;
  R3D_CUDA_TRY(ctx, mem.alloc(&s.Lm, ((size_t)nB + 1) * nB + 64));
  R3D_CUDA_TRY(ctx, mem.alloc(&s.Linv, (size_t)chol_blocks * r3d::ba::NB * r3d::ba::NB));
  // Envelope of the reduced system at tile granularity (the union over ranks: every rank factors the summed S)
  const int ntr = (nB + 1 + r3d::ba::NB - 1) / r3d::ba::NB;
  std::vector<double> fc(p->n_cams);
  for (uint32_t c = 0; c < p->n_cams; ++c) fc[c] = -(double)plan.first_cam[c];
  if (ctx->comm_world > 1 && p->n_cams) {  // min over ranks = -max(-x)
    double* d_fc = nullptr;
    R3D_CUDA_TRY(ctx, mem.alloc(&d_fc, p->n_cams));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_fc, fc.data(), (size_t)p->n_cams * 8, cudaMemcpyHostToDevice, w.stream));
    if ((rc = comm_allreduce(ctx, w.stream, d_fc, p->n_cams, kCommMax))) return rc;
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(fc.data(), d_fc, (size_t)p->n_cams * 8, cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  }
  std::vector<int> ft(ntr, 0);
  for (int ti = 0; ti < ntr; ++ti) {
    int first = ti * r3d::ba::NB;
    for (int r = ti * r3d::ba::NB; r < std::min((ti + 1) * r3d::ba::NB, nB + 1); ++r) {
      const int fcol = r < 6 * (int)p->n_cams ? 6 * (int)(-fc[r / 6]) : 0;  // intrinsics rows, rhs row: from column 0
      first = std::min(first, fcol);
    }
    ft[ti] = first / r3d::ba::NB;
  }
  // per panel: active row tiles -> tile pairs; compare with the dense kernel's two grid barriers + full trailing update
  {
    const char* e = getenv("R3D_BA_ENV_CTAS");
    if (e && atoi(e) >= 1 && atoi(e) <= r3d::ba::kEnvMaxCluster) s.env_ctas = atoi(e);
  }
  int max_act = 0;
  double est_env = 0.0, est_dense = 0.0;
  for (int k = 0; k < chol_blocks; ++k) {
    int act = 0;
    for (int ti = k + 1; ti < ntr; ++ti) act += ft[ti] <= k;
    max_act = std::max(max_act, act);
    est_env += 32.0 + 5.0 * std::ceil((double)(act * (act + 1) / 2) / (16.0 * s.env_ctas)) + 0.6 * act;
    const int rem = ntr - k - 1;
    est_dense += 20.0 + 3.0 * std::ceil((double)(rem * (rem + 1) / 2) / (4.0 * w.sm_count));
  }
  // Measured at C5 (profiles/r02_ba_cholesky_ab.md): the envelope kernel does 7x fewer tile products but its panels
  // cost 54 us on 8 SMs (register potrf 8, redundant trsm 10 -- shared-memory instruction issue --, fp64 syrk on 8 SMs
  // 20, cluster barrier 14) against 29 us for the dense cooperative kernel on 148 SMs, so the dense kernel stays the
  // default; R3D_BA_CHOL=envelope selects the envelope kernel where it applies (A/B and tests), =auto trusts the
  // estimate.
  s.use_env = false;
  if (chol == kCholAuto) s.use_env = max_act <= r3d::ba::kEnvMaxActive && est_env < est_dense;
  if (chol == kCholEnvelope) s.use_env = max_act <= r3d::ba::kEnvMaxActive;
  if (s.use_env) {
    R3D_CUDA_TRY(ctx, mem.alloc(&s.ft, (size_t)ntr));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(s.ft, ft.data(), (size_t)ntr * sizeof(int), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));  // ft is a local
  }
  static const bool dbg = getenv("R3D_DEBUG_TIMING") != nullptr;
  if (dbg) fprintf(stderr, "[r3d] BA linear solve: %s (n = %d, %d tiles, <= %d active row tiles per panel, estimate %.0f vs %.0f us dense)\n",
                   s.use_env ? "envelope Cholesky, one cluster" : "dense cooperative Cholesky", nB, ntr, max_act, est_env, est_dense);
  return R3D_OK;
}

int read_scal(r3d_ctx* ctx, DeviceWorker& w, const Dev& d, double* h_scal) {
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(h_scal, d.scal, 8 * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  return R3D_OK;
}

// gradient + diag at the current parameters (scaled; the Jacobi scaling itself is made from this diag when
// make_scale), and the largest unscaled gradient component
int ba_evaluate(r3d_ctx* ctx, DeviceWorker& w, const Dev& d, bool make_scale, double* gmax) {
  int rc;
  const size_t nparam = (size_t)d.nB + 3 * (size_t)d.n_pts;
  const int nB = (int)d.nB;
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d.gu, 0, nparam * 8, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d.du, 0, nparam * 8, w.stream));
  r3d::ba::k_ba_eval<<<w.sm_count * 8, 256, 0, w.stream>>>(d);
  if (d.n_priors && d.owns_shared) r3d::ba::k_ba_priors<<<(d.n_priors + 127) / 128, 128, 0, w.stream>>>(d, d.poses, 1, nullptr);
  // camera / intrinsic gradient and column norms are sums over every rank's observations
  if ((rc = comm_allreduce(ctx, w.stream, d.gu, nB, kCommSum))) return rc;
  if ((rc = comm_allreduce(ctx, w.stream, d.du, nB, kCommSum))) return rc;
  if (make_scale) r3d::ba::k_ba_make_scale<<<(unsigned)((nparam + 255) / 256), 256, 0, w.stream>>>(d.scale, d.du, nparam);
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d.scal + 5, 0, sizeof(double), w.stream));
  r3d::ba::k_ba_apply_scale<<<(unsigned)((nparam + 255) / 256), 256, 0, w.stream>>>(d.scale, d.gu, d.du, d.g, d.diag, nparam, d.scal + 5);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  if ((rc = comm_allreduce(ctx, w.stream, d.scal + 5, 1, kCommMax))) return rc;
  double h_scal[8];
  if ((rc = read_scal(ctx, w, d, h_scal))) return rc;
  *gmax = h_scal[5];
  return R3D_OK;
}

// One LM step at trust-region radius 1 / inv_radius: the reduced camera system S | rhs (Schur kernels, prior U blocks,
// k_ba_finish_S), its Cholesky solve, the point back-substitution and the candidate parameters; d.scal[1..4] =
// 2 * model cost change, |dx|^2, |x|^2, not-PD flag.  S_copy (nB * nB + nB, or nullptr) receives S | rhs before the
// factorisation overwrites it.
int ba_step(r3d_ctx* ctx, DeviceWorker& w, const Dev& d, const StepPlan& s, double inv_radius, double* S_copy) {
  int rc;
  const int nB = (int)d.nB;
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d.S, 0, ((size_t)nB * nB + nB) * 8, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d.scal, 0, 5 * sizeof(double), w.stream));
  if (s.plan.n_batches)
    r3d::ba::k_ba_schur_batched<<<s.plan.n_batches, 256, r3d::ba::kBatchSmemBytes, w.stream>>>(d, s.plan.t, inv_radius);
  if (s.plan.n_long)  // long tracks and whatever else the batched kernel cannot take
    r3d::ba::k_ba_schur_cta<<<s.long_grid, r3d::ba::kCtaThreads, 0, w.stream>>>(d, s.plan.d_long, s.plan.n_long, inv_radius,
                                                                               s.long_scr, s.long_cols, s.plan.long_cap);
  if (d.n_priors && d.owns_shared) r3d::ba::k_ba_priors<<<(d.n_priors + 127) / 128, 128, 0, w.stream>>>(d, d.poses, 2, nullptr);
  // the exchange step: partial reduced camera systems of the point partitions -> their sum (NVLink)
  if ((rc = comm_allreduce(ctx, w.stream, d.S, (size_t)nB * nB + nB, kCommSum))) return rc;
  {
    dim3 b(32, 8), g((nB + 31) / 32, (nB + 7) / 8);
    r3d::ba::k_ba_finish_S<<<g, b, 0, w.stream>>>(d, inv_radius);
  }
  if (S_copy)
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(S_copy, d.S, ((size_t)nB * nB + nB) * 8, cudaMemcpyDeviceToDevice, w.stream));
  if (s.use_env) {
    if ((rc = envelope_cholesky(ctx, w, d.S, s.Lm, nB, s.ft, s.env_ctas, d.scal + 4, d.delta))) return rc;
  } else {
    if ((rc = dense_cholesky(ctx, w, d.S, s.Lm, s.Linv, nB, d.scal + 4, d.delta))) return rc;
  }
  r3d::ba::k_ba_backsub<<<(d.n_pts + 127) / 128, 128, 0, w.stream>>>(d, inv_radius);
  r3d::ba::k_ba_update<<<w.sm_count * 4, 256, 0, w.stream>>>(d, inv_radius);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return comm_allreduce(ctx, w.stream, d.scal + 1, 3, kCommSum);
}

}  // namespace

extern "C" {

void r3d_ba_default_options(r3d_ba_options* o) {
  if (!o) return;
  o->max_iterations = 500;      // OpenMVG: ceres_options.max_num_iterations = 500
  o->huber_a = 16.0;            // new ceres::HuberLoss(Square(4.0))
  o->refine_intrinsics = 1;     // Intrinsic_Parameter_Type::ADJUST_ALL
  o->function_tolerance = 1e-6; // Ceres defaults
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
  o->initial_radius = 1e4;
  o->prior_huber_a = 0.0;       // trivial loss unless the caller passes the registration's robust fitting error
}

int r3d_ba_residuals(r3d_ctx* ctx, const r3d_ba_problem* p, double* res) {
  if (!ctx || !p || !res) return fail(ctx, R3D_ERR_INVALID, "r3d_ba_residuals: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  DeviceArrays mem;
  mem.w = &w;
  Dev d;
  int rc = setup_problem(ctx, w, p, mem, d, false, 0.0, false);
  if (rc) return rc;
  double* dres;
  R3D_CUDA_TRY(ctx, mem.alloc(&dres, 2 * p->n_obs));
  r3d::ba::k_ba_abs_residuals<<<w.sm_count * 4, 256, 0, w.stream>>>(d, dres);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(res, dres, 2 * p->n_obs * 8, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  return R3D_OK;
}

int r3d_bundle_adjust(r3d_ctx* ctx, r3d_ba_problem* p, const r3d_ba_options* opt, r3d_ba_summary* sum, double* cost_trace) {
  if (!ctx || !p || !opt || !sum) return fail(ctx, R3D_ERR_INVALID, "r3d_bundle_adjust: bad arguments");
  const auto t_begin = std::chrono::steady_clock::now();
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  DeviceArrays mem;
  mem.w = &w;
  Dev d;
  StepPlan sp;
  static const bool per_point_schur = getenv("R3D_BA_SCHUR") && std::string(getenv("R3D_BA_SCHUR")) == "point";
  sp.plan.want_batched = !per_point_schur;
  int rc = setup_problem(ctx, w, p, mem, d, opt->refine_intrinsics != 0, opt->huber_a, true, nullptr, &sp.plan);
  if (rc) return rc;
  d.prior_huber_a = opt->prior_huber_a;
  {
    const char* force = getenv("R3D_BA_CHOL");
    const CholChoice chol = !force ? kCholDense : std::string(force) == "auto" ? kCholAuto
                          : std::string(force) == "envelope" ? kCholEnvelope : kCholDense;
    if ((rc = setup_step(ctx, w, p, mem, d, chol, sp))) return rc;
  }
  sum->seconds_setup = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  const int grid_obs = w.sm_count * 8;
  double h_scal[8];
  auto eval_cost = [&](const double* poses, const double* intr, const double* pts, double* out) -> int {
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d.scal, 0, sizeof(double), w.stream));
    r3d::ba::k_ba_cost<<<grid_obs, 256, 0, w.stream>>>(d, poses, intr, pts, d.scal);
    if (d.n_priors && d.owns_shared)  // camera-only blocks: counted once across ranks
      r3d::ba::k_ba_priors<<<(d.n_priors + 127) / 128, 128, 0, w.stream>>>(d, poses, 0, d.scal);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    if ((rc = comm_allreduce(ctx, w.stream, d.scal, 1, kCommSum))) return rc;
    if ((rc = read_scal(ctx, w, d, h_scal))) return rc;
    *out = h_scal[0];
    return R3D_OK;
  };
  double gmax = 0;

  double cost = 0;
  if ((rc = eval_cost(d.poses, d.intr, d.pts, &cost))) return rc;
  sum->initial_cost = cost;
  sum->seconds_linear = 0;
  if (cost_trace) cost_trace[0] = cost;
  r3d::LmTrustRegion lm(r3d::lm_params(*opt));
  if ((rc = ba_evaluate(ctx, w, d, true, &gmax))) return rc;  // the Jacobi scaling is fixed at the initial parameters
  const bool stop = lm.start(gmax);
  for (uint32_t iter = 1; !stop && iter <= opt->max_iterations; ++iter) {
    lm.iterations = iter;
    const auto t_lin = std::chrono::steady_clock::now();
    if ((rc = ba_step(ctx, w, d, sp, 1.0 / lm.radius, nullptr))) return rc;
    if ((rc = read_scal(ctx, w, d, h_scal))) return rc;
    sum->seconds_linear += std::chrono::duration<double>(std::chrono::steady_clock::now() - t_lin).count();
    const double model_cost_change = 0.5 * h_scal[1];
    bool accepted = false;
    if (lm.step_usable(h_scal[4] == 0.0, model_cost_change)) {
      if (lm.step_too_small(h_scal[2], h_scal[3])) {
        if (cost_trace) cost_trace[iter] = cost;
        break;
      }
      double new_cost = 0;
      if ((rc = eval_cost(d.poses_new, d.intr_new, d.pts_new, &new_cost))) return rc;
      if ((accepted = lm.accept(cost, new_cost, model_cost_change))) {
        std::swap(d.poses, d.poses_new);
        std::swap(d.intr, d.intr_new);
        std::swap(d.pts, d.pts_new);
        cost = new_cost;
        if (cost_trace) cost_trace[iter] = cost;
        if ((rc = ba_evaluate(ctx, w, d, false, &gmax))) return rc;
        if (lm.converged(gmax)) break;
      }
    }
    if (!accepted) {
      if (cost_trace) cost_trace[iter] = cost;
      if (lm.reject()) break;
    }
  }
  sum->iterations = lm.iterations;
  sum->successful_steps = lm.successful;
  sum->termination = lm.termination;
  sum->final_cost = cost;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(p->poses, d.poses, 6 * (size_t)p->n_cams * 8, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(p->intrinsics, d.intr, 6 * (size_t)p->n_intr * 8, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(p->points, d.pts, 3 * (size_t)p->n_pts * 8, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  sum->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  return R3D_OK;
}

int r3d_debug_ba_step(r3d_ctx* ctx, const r3d_ba_problem* p, const r3d_ba_options* opt, double radius, int schur_route,
                      int chol_method, r3d_ba_step_out* out) {
  if (!ctx || !p || !opt || !out || !(radius > 0.0) || (schur_route != 0 && schur_route != 1) || (chol_method != 0 && chol_method != 1))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_ba_step: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  DeviceArrays mem;
  mem.w = &w;
  Dev d;
  StepPlan sp;
  sp.plan.want_batched = schur_route == 0;
  int rc = setup_problem(ctx, w, p, mem, d, opt->refine_intrinsics != 0, opt->huber_a, true, nullptr, &sp.plan);
  if (rc) return rc;
  d.prior_huber_a = opt->prior_huber_a;
  if ((rc = setup_step(ctx, w, p, mem, d, chol_method ? kCholEnvelope : kCholDense, sp))) return rc;
  if (chol_method && !sp.use_env) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_ba_step: the envelope kernel does not take this system");
  const size_t nB = d.nB, nparam = nB + 3 * (size_t)d.n_pts;
  double* S_copy;
  R3D_CUDA_TRY(ctx, mem.alloc(&S_copy, nB * nB + nB));
  double gmax = 0.0;
  if ((rc = ba_evaluate(ctx, w, d, true, &gmax))) return rc;
  if ((rc = ba_step(ctx, w, d, sp, 1.0 / radius, S_copy))) return rc;
  double h_scal[8];
  if ((rc = read_scal(ctx, w, d, h_scal))) return rc;
  const std::pair<double*, const double*> arrays[] = {{out->g, d.g}, {out->diag, d.diag}, {out->scale, d.scale}, {out->delta, d.delta}};
  for (const auto& a : arrays)
    if (a.first) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(a.first, a.second, nparam * 8, cudaMemcpyDeviceToHost, w.stream));
  if (out->S) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(out->S, S_copy, nB * nB * 8, cudaMemcpyDeviceToHost, w.stream));
  if (out->rhs) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(out->rhs, S_copy + nB * nB, nB * 8, cudaMemcpyDeviceToHost, w.stream));
  if (out->Vinv) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(out->Vinv, d.Vinv, 9 * (size_t)d.n_pts * 8, cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  out->nB = d.nB;
  out->n_batches = sp.plan.n_batches;
  out->n_long = sp.plan.n_long;
  out->not_pd = h_scal[4] != 0.0;
  out->gmax = gmax;
  out->model_cost_change = 0.5 * h_scal[1];
  out->dx_norm2 = h_scal[2];
  out->x_norm2 = h_scal[3];
  return R3D_OK;
}

int r3d_debug_cholesky(r3d_ctx* ctx, int method, int n, const double* A, const int* ft, int grid, double* L_out, double* x_out,
                       double* Linv_out, int* not_pd) {
  if (!ctx || !A || !L_out || !x_out || !not_pd || n < 1 || (method != 0 && method != 1) || grid < 0)
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_cholesky: bad arguments");
  const int NB = r3d::ba::NB;
  const int nblk = (n + NB - 1) / NB, ntr = (n + 1 + NB - 1) / NB;
  if (method == 1) {  // everything the envelope kernel assumes, before anything reaches the device
    if (n % 2) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_cholesky: the envelope kernel needs an even n");
    if (!ft || grid > r3d::ba::kEnvMaxCluster) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_cholesky: bad ft / cluster size");
    for (int t = 0; t < ntr; ++t)
      if (ft[t] < 0 || ft[t] > t) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_cholesky: ft[" + std::to_string(t) + "] outside 0.." + std::to_string(t));
    for (int k = 0; k < nblk; ++k) {
      int act = 0;
      for (int ti = k + 1; ti < ntr; ++ti) act += ft[ti] <= k;
      if (act > r3d::ba::kEnvMaxActive)
        return fail(ctx, R3D_ERR_INVALID, "r3d_debug_cholesky: panel " + std::to_string(k) + " has " + std::to_string(act) + " active row tiles");
    }
  }
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  int rc;
  if (method == 0 && (rc = dense_cholesky_grid(ctx, w, &grid))) return rc;
  DeviceArrays mem;
  mem.w = &w;
  const size_t nA = (size_t)(n + 1) * n;
  double *dA, *dL, *dLinv, *dx, *dflag;
  int* dft = nullptr;
  // as r3d_bundle_adjust allocates S | rhs and Lm: 64 doubles of slack that k_chol_envelope reads past row n
  R3D_CUDA_TRY(ctx, mem.alloc(&dA, nA + 64));
  R3D_CUDA_TRY(ctx, mem.alloc(&dL, nA + 64));
  R3D_CUDA_TRY(ctx, mem.alloc(&dLinv, (size_t)nblk * NB * NB));
  R3D_CUDA_TRY(ctx, mem.alloc(&dx, (size_t)n));
  R3D_CUDA_TRY(ctx, mem.alloc(&dflag, 1));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(dA, A, nA * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(dA + nA, 0, 64 * sizeof(double), w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(dL, 0, (nA + 64) * sizeof(double), w.stream));  // the upper triangle comes back as 0
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(dLinv, 0, (size_t)nblk * NB * NB * sizeof(double), w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(dflag, 0, sizeof(double), w.stream));
  if (method == 0) {
    if ((rc = dense_cholesky(ctx, w, dA, dL, dLinv, n, dflag, dx, grid))) return rc;
  } else {
    R3D_CUDA_TRY(ctx, mem.alloc(&dft, (size_t)ntr));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(dft, ft, (size_t)ntr * sizeof(int), cudaMemcpyHostToDevice, w.stream));
    if ((rc = envelope_cholesky(ctx, w, dA, dL, n, dft, grid ? grid : r3d::ba::kEnvMaxCluster, dflag, dx))) return rc;
  }
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  double flag = 0.0;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(L_out, dL, nA * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(x_out, dx, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  if (Linv_out && method == 0)
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(Linv_out, dLinv, (size_t)nblk * NB * NB * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(&flag, dflag, sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  *not_pd = flag != 0.0;
  return R3D_OK;
}

}  // extern "C"
