// relpose.cu -- relative pose of every image pair (r3d_relative_poses).
// COMPILED WITH --fmad=false (regard3d_b200/build.py): the cheirality counts and the chosen motion must equal the CPU
// restatement's (oracle/oracle_relpose.cpp) bit for bit, and the two-view bundle adjustment follows its LM decisions.
//
// Replaces the loop body of GlobalSfMReconstructionEngine_RelativeMotions::Compute_Relative_Rotations (OpenMVG 1.4,
// reached from src/threads/R3DTriangulationThread.cpp:201-250).  Three stages, each one CTA per pair:
//   1. robustRelativePose's AC-RANSAC: the essential filter's persistent kernel (k_acransac_fused<2>, acransac_host.cu)
//      with the relative-pose precision and budget; it also hands back the best model F = K2^-T E K1^-1 and errorMax;
//   2. k_relpose_cheirality: E = K2^T F K1 (the 5-point solver's E up to rounding), MotionFromEssential
//      (relpose_math.cuh) and the DLT depth test of every inlier under the four motions, strided over the threads;
//      the first motion with the most points in front of both cameras;
//   3. k_relpose_ba: the whole Levenberg-Marquardt solve of oracle_ba.cpp on the pair's two-view scene (both poses,
//      one DLT point per match, intrinsics fixed, Huber loss): Jacobi scaling, the D^2 clamp and radius rules, Schur
//      elimination of the points into the 12 x 12 camera system, Cholesky, the trial cost and Ceres' termination
//      tests.  Per-point state lives in a global scratch slot of the CTA (structure of arrays, mostly L2-resident);
//      the camera system and the state machine live in shared memory.  Every reduction has a fixed order, so a call
//      is reproducible.  FP64 throughout; the kernel is bound by FP64 latency, not by tensor cores or HBM.
#include "acransac.cuh"
#include "ba_model.cuh"
#include "lm_trust_region.cuh"
#include "relpose_math.cuh"

#include <cstring>
#include <numeric>

namespace r3d {

namespace {

struct RpPair {            // a pair that reached the cheirality stage
  uint32_t in_ofs, n_in;   // its AC-RANSAC inliers in x_in1 / x_in2 (residual order)
  uint32_t all_ofs, M;     // every match of the pair in x_all1 / x_all2 (bundle adjustment)
  double K[6];             // f, ppx, ppy of I, then of J
  double F[9];             // AC-RANSAC's best model
};

struct RpCheir {           // cheirality result
  double E[9];
  double R[9], t[3];
  uint32_t cnt[4];
  int best;
  int pad_;
};

struct RpBa {              // bundle adjustment: initial state in, solution out
  double pose[12];         // angle-axis | t of camera I, then of J
  double R[9], t[3];       // the chosen motion (initial triangulation)
  uint32_t iterations, successful;
  int termination;
  int pad_;
  double initial_cost, final_cost;
};

constexpr int kCThreads = 128;

__global__ void __launch_bounds__(kCThreads) k_relpose_cheirality(const RpPair* __restrict__ pairs, const double2* __restrict__ x1,
                                                                   const double2* __restrict__ x2, RpCheir* __restrict__ out) {
  __shared__ double Rs[36], ts[12], P2[48], E[9];
  __shared__ uint32_t cnt[4];
  const RpPair pr = pairs[blockIdx.x];
  if (threadIdx.x == 0) {
    rp::essential_from_fundamental(pr.F, pr.K, pr.K + 3, E);
    rp::motions_from_essential(E, Rs, ts);
    for (int k = 0; k < 4; ++k) {
      rp::rt_matrix(Rs + 9 * k, ts + 3 * k, P2 + 12 * k);
      cnt[k] = 0;
    }
  }
  __syncthreads();
  uint32_t c[4] = {0, 0, 0, 0};
  for (uint32_t i = threadIdx.x; i < pr.n_in; i += kCThreads) {
    const double2 a = x1[pr.in_ofs + i], b = x2[pr.in_ofs + i];
    double b1[3], b2[3];
    rp::bearing_vec(pr.K, a.x, a.y, b1);
    rp::bearing_vec(pr.K + 3, b.x, b.y, b2);
    for (int k = 0; k < 4; ++k) c[k] += rp::in_front(P2 + 12 * k, b1, b2) ? 1u : 0u;
  }
  for (int k = 0; k < 4; ++k) {
    uint32_t v = c[k];
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31u) == 0 && v) atomicAdd(&cnt[k], v);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    for (int k = 1; k < 4; ++k)
      if (cnt[k] > cnt[best]) best = k;  // std::max_element: the first maximum
    RpCheir o;
    for (int i = 0; i < 9; ++i) o.E[i] = E[i];
    for (int i = 0; i < 9; ++i) o.R[i] = Rs[9 * best + i];
    for (int i = 0; i < 3; ++i) o.t[i] = ts[3 * best + i];
    for (int k = 0; k < 4; ++k) o.cnt[k] = cnt[k];
    o.best = best;
    o.pad_ = 0;
    out[blockIdx.x] = o;
  }
}

// ---- two-view Levenberg-Marquardt --------------------------------------------------------------------------------
constexpr int kBThreads = 256;
constexpr int kBWarps = kBThreads / 32;
constexpr int kEntries = 90;             // 78 lower-triangle entries of the 12 x 12 camera system + 12 right-hand sides
constexpr int kMaxGroups = 8;            // point ranges of one fixed-order entry reduction
// per-point fields of the scratch slot (structure of arrays: field f of point p at f * cap + p)
constexpr int fX = 0;                    // 2 x 3: current and trial point (double-buffered)
constexpr int fR = 6;                    // 4: scaled residuals, observation I then J
constexpr int fJc = 10;                  // 24: scaled pose Jacobians, 2 x 6 per observation
constexpr int fJp = 34;                  // 12: scaled point Jacobians, 2 x 3 per observation
constexpr int fS = 46;                   // 3: Jacobi scale of the point's columns
constexpr int fG = 49;                   // 3: gradient
constexpr int fD = 52;                   // 3: diag(J^T J)
constexpr int fDel = 55;                 // 3: step
constexpr int fVi = 58;                  // 9: (V + D^2)^-1
constexpr int fWV = 67;                  // 36: W (V + D^2)^-1, 12 x 3
constexpr int fVg = 103;                 // 3: (V + D^2)^-1 g
constexpr int kFields = 106;

struct BaSmem {
  double pose[12], pose_new[12], scale[12], g[12], diag[12], D2[12], delta[12];
  double S[144], rhs[12];
  double part[kMaxGroups * kEntries];
  double sums[kEntries];
  double red[kBWarps];
  double P1[12], P2[12];
  double intr[2][6];
  int pd;
  uint32_t work;
};

// sums[e] = sum over the points of fn(e, p), e < n: the points are cut into fixed ranges, one thread per (range,
// entry) walks its range in order, the ranges are added in order -- the same bits on every call
template <class Fn>
__device__ void entry_sums(int n, uint32_t N, BaSmem& S, Fn fn) {
  int groups = kBThreads / n;
  if (groups > kMaxGroups) groups = kMaxGroups;
  const int e = (int)threadIdx.x % n, g = (int)threadIdx.x / n;
  if (g < groups) {
    const uint32_t chunk = (N + groups - 1) / groups;
    const uint32_t p0 = min(N, (uint32_t)g * chunk), p1 = min(N, p0 + chunk);
    double s = 0.0;
    for (uint32_t p = p0; p < p1; ++p) s += fn(e, p);
    S.part[g * kEntries + e] = s;
  }
  __syncthreads();
  if ((int)threadIdx.x < n) {
    double s = 0.0;
    for (int q = 0; q < groups; ++q) s += S.part[q * kEntries + threadIdx.x];
    S.sums[threadIdx.x] = s;
  }
  __syncthreads();
}

// one persistent CTA per pair; order: pair ids, most matches first; scratch: kFields x cap doubles per CTA
__global__ void __launch_bounds__(kBThreads) k_relpose_ba(const RpPair* __restrict__ pairs, const uint32_t* __restrict__ order,
                                                          uint32_t n_order, uint32_t* __restrict__ work_counter,
                                                          const double2* __restrict__ xa1, const double2* __restrict__ xa2,
                                                          RpBa* __restrict__ io, LmParams prm, double* __restrict__ scratch,
                                                          uint32_t cap) {
  __shared__ BaSmem S;
  const uint32_t tid = threadIdx.x;
  double* buf = scratch + (size_t)blockIdx.x * kFields * cap;
#define F(f, p) buf[(size_t)(f) * cap + (p)]
  for (;;) {
    __syncthreads();
    if (tid == 0) S.work = atomicAdd(work_counter, 1u);
    __syncthreads();
    const uint32_t wk = S.work;
    if (wk >= n_order) break;
    const uint32_t pid = order[wk];
    const RpPair pr = pairs[pid];
    const uint32_t N = pr.M;
    const double2* o1 = xa1 + pr.all_ofs;
    const double2* o2 = xa2 + pr.all_ofs;
    if (tid < 12) S.pose[tid] = io[pid].pose[tid];
    if (tid < 12) {  // K [I | 0] and K [R | t]
      const double Id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z[3] = {0, 0, 0};
      if (tid == 0) rp::projective(pr.K, Id, z, S.P1);
      if (tid == 1) rp::projective(pr.K + 3, io[pid].R, io[pid].t, S.P2);
      if (tid < 2)
        for (int k = 0; k < 6; ++k) S.intr[tid][k] = k < 3 ? pr.K[3 * tid + k] : 0.0;
    }
    __syncthreads();
    int cur = 0;  // which half of the point double buffer holds the current points
    for (uint32_t p = tid; p < N; p += kBThreads) {
      const double2 a = o1[p], b = o2[p];
      const double h1[3] = {a.x, a.y, 1.0}, h2[3] = {b.x, b.y, 1.0};
      double X[3];
      rp::triangulate2(S.P1, h1, S.P2, h2, X);
      for (int i = 0; i < 3; ++i) F(fX + i, p) = X[i];
    }
    __syncthreads();

    // total cost at (poses, points half h): sum of 1/2 rho(|r|^2) over both observations of every point
    auto total_cost = [&](const double* pose, int h) -> double {
      double c = 0.0;
      for (uint32_t p = tid; p < N; p += kBThreads) {
        const double X[3] = {F(fX + 3 * h, p), F(fX + 3 * h + 1, p), F(fX + 3 * h + 2, p)};
        for (int v = 0; v < 2; ++v) {
          const double2 ob = v ? o2[p] : o1[p];
          double r[2], rho1;
          ba::residual_only(3, S.intr[v], nullptr, pose + 6 * v, X, ob.x, ob.y, r);
          c += 0.5 * ba::huber_rho(r[0] * r[0] + r[1] * r[1], prm.huber_a, &rho1);
        }
      }
      return block_sum_fixed<kBThreads>(c, S.red);
    };
    // residuals, Jacobians (Corrector-scaled), the Jacobi scale on the first call, then g and diag(J^T J)
    auto evaluate = [&](bool first) {
      for (uint32_t p = tid; p < N; p += kBThreads) {
        const double X[3] = {F(fX + 3 * cur, p), F(fX + 3 * cur + 1, p), F(fX + 3 * cur + 2, p)};
        for (int v = 0; v < 2; ++v) {
          const double2 ob = v ? o2[p] : o1[p];
          double r[2], Ji[12], Jc[12], Jp[6], rho1;
          ba::residual_jacobian(3, S.intr[v], nullptr, S.pose + 6 * v, X, ob.x, ob.y, r, Ji, Jc, Jp);
          ba::huber_rho(r[0] * r[0] + r[1] * r[1], prm.huber_a, &rho1);
          const double sq = sqrt(rho1);
          for (int a = 0; a < 2; ++a) F(fR + 2 * v + a, p) = r[a] * sq;
          for (int k = 0; k < 12; ++k) F(fJc + 12 * v + k, p) = Jc[k] * sq;
          for (int k = 0; k < 6; ++k) F(fJp + 6 * v + k, p) = Jp[k] * sq;
        }
        if (first) {
          for (int i = 0; i < 3; ++i) {
            double n2 = 0.0;
            for (int v = 0; v < 2; ++v)
              for (int a = 0; a < 2; ++a) n2 += F(fJp + 6 * v + 3 * a + i, p) * F(fJp + 6 * v + 3 * a + i, p);
            F(fS + i, p) = 1.0 / (1.0 + sqrt(n2));
          }
        }
      }
      __syncthreads();
      if (first) {  // camera columns: 1 / (1 + ||column||)
        entry_sums(12, N, S, [&](int e, uint32_t p) {
          const int v = e / 6, k = e % 6;
          const double j0 = F(fJc + 12 * v + k, p), j1 = F(fJc + 12 * v + 6 + k, p);
          return j0 * j0 + j1 * j1;
        });
        if (tid < 12) S.scale[tid] = 1.0 / (1.0 + sqrt(S.sums[tid]));
        __syncthreads();
      }
      for (uint32_t p = tid; p < N; p += kBThreads) {  // apply the scaling; point gradient and diagonal
        double gp[3] = {0, 0, 0}, dp[3] = {0, 0, 0};
        const double sp[3] = {F(fS, p), F(fS + 1, p), F(fS + 2, p)};
        for (int v = 0; v < 2; ++v)
          for (int a = 0; a < 2; ++a) {
            const double ra = F(fR + 2 * v + a, p);
            for (int k = 0; k < 6; ++k) F(fJc + 12 * v + 6 * a + k, p) *= S.scale[6 * v + k];
            for (int k = 0; k < 3; ++k) {
              const double j = F(fJp + 6 * v + 3 * a + k, p) * sp[k];
              F(fJp + 6 * v + 3 * a + k, p) = j;
              gp[k] += j * ra;
              dp[k] += j * j;
            }
          }
        for (int k = 0; k < 3; ++k) { F(fG + k, p) = gp[k]; F(fD + k, p) = dp[k]; }
      }
      __syncthreads();
      entry_sums(24, N, S, [&](int e, uint32_t p) {  // camera gradient (e < 12) and diagonal
        const int c = e % 12, v = c / 6, k = c % 6;
        const double j0 = F(fJc + 12 * v + k, p), j1 = F(fJc + 12 * v + 6 + k, p);
        return e < 12 ? j0 * F(fR + 2 * v, p) + j1 * F(fR + 2 * v + 1, p) : j0 * j0 + j1 * j1;
      });
      if (tid < 12) { S.g[tid] = S.sums[tid]; S.diag[tid] = S.sums[12 + tid]; }
      __syncthreads();
    };
    auto grad_max = [&]() -> double {
      double m = 0.0;
      for (uint32_t p = tid; p < N; p += kBThreads)
        for (int k = 0; k < 3; ++k) m = fmax(m, fabs(F(fG + k, p) / F(fS + k, p)));
      m = block_max_fixed<kBThreads>(m, S.red);
      for (int j = 0; j < 12; ++j) m = fmax(m, fabs(S.g[j] / S.scale[j]));
      return m;
    };

    double cost = total_cost(S.pose, cur);
    const double initial_cost = cost;
    LmTrustRegion lm(prm);  // every thread keeps its own: the inputs are block-wide, so are the decisions
    evaluate(true);
    if (!lm.start(grad_max()))
      for (uint32_t iter = 1; iter <= prm.max_iterations; ++iter) {
        lm.iterations = iter;
        // LevenbergMarquardtStrategy: D^2 = clamp(diag(J^T J), 1e-6, 1e32) / radius
        if (tid < 12) S.D2[tid] = fmin(fmax(S.diag[tid], 1e-6), 1e32) / lm.radius;
        for (uint32_t p = tid; p < N; p += kBThreads) {  // point blocks: (V + D^2)^-1, W (V + D^2)^-1, (V + D^2)^-1 g
          double V[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
          for (int v = 0; v < 2; ++v)
            for (int a = 0; a < 2; ++a)
              for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) V[3 * i + j] += F(fJp + 6 * v + 3 * a + i, p) * F(fJp + 6 * v + 3 * a + j, p);
          for (int i = 0; i < 3; ++i) V[4 * i] += fmin(fmax(F(fD + i, p), 1e-6), 1e32) / lm.radius;
          const double c00 = V[4] * V[8] - V[5] * V[7], c01 = V[5] * V[6] - V[3] * V[8], c02 = V[3] * V[7] - V[4] * V[6];
          const double det = V[0] * c00 + V[1] * c01 + V[2] * c02;
          double Vi[9];
          Vi[0] = c00 / det; Vi[1] = (V[2] * V[7] - V[1] * V[8]) / det; Vi[2] = (V[1] * V[5] - V[2] * V[4]) / det;
          Vi[3] = c01 / det; Vi[4] = (V[0] * V[8] - V[2] * V[6]) / det; Vi[5] = (V[2] * V[3] - V[0] * V[5]) / det;
          Vi[6] = c02 / det; Vi[7] = (V[1] * V[6] - V[0] * V[7]) / det; Vi[8] = (V[0] * V[4] - V[1] * V[3]) / det;
          const double g0 = F(fG, p), g1 = F(fG + 1, p), g2 = F(fG + 2, p);
          for (int i = 0; i < 9; ++i) F(fVi + i, p) = Vi[i];
          for (int i = 0; i < 3; ++i) F(fVg + i, p) = Vi[3 * i] * g0 + Vi[3 * i + 1] * g1 + Vi[3 * i + 2] * g2;
          for (int v = 0; v < 2; ++v)
            for (int i = 0; i < 6; ++i) {
              double W[3];
              for (int j = 0; j < 3; ++j)
                W[j] = F(fJc + 12 * v + i, p) * F(fJp + 6 * v + j, p) + F(fJc + 12 * v + 6 + i, p) * F(fJp + 6 * v + 3 + j, p);
              for (int j = 0; j < 3; ++j) F(fWV + 3 * (6 * v + i) + j, p) = W[0] * Vi[j] + W[1] * Vi[3 + j] + W[2] * Vi[6 + j];
            }
        }
        __syncthreads();
        // reduced camera system S = U + D^2 - W V^-1 W^T (lower triangle) and rhs = -g + W V^-1 g_p
        entry_sums(kEntries, N, S, [&](int e, uint32_t p) {
          auto Wel = [&](int b, int i) {  // W[b][i] of this point
            const int v = b / 6, k = b % 6;
            return F(fJc + 12 * v + k, p) * F(fJp + 6 * v + i, p) + F(fJc + 12 * v + 6 + k, p) * F(fJp + 6 * v + 3 + i, p);
          };
          if (e >= 78) {
            const int a = e - 78;
            return Wel(a, 0) * F(fVg, p) + Wel(a, 1) * F(fVg + 1, p) + Wel(a, 2) * F(fVg + 2, p);
          }
          int a = 0;
          while ((a + 1) * (a + 2) / 2 <= e) ++a;
          const int b = e - a * (a + 1) / 2;
          double u = 0.0;
          if (a / 6 == b / 6) {
            const int v = a / 6, ka = a % 6, kb = b % 6;
            u = F(fJc + 12 * v + ka, p) * F(fJc + 12 * v + kb, p) + F(fJc + 12 * v + 6 + ka, p) * F(fJc + 12 * v + 6 + kb, p);
          }
          const double s = F(fWV + 3 * a, p) * Wel(b, 0) + F(fWV + 3 * a + 1, p) * Wel(b, 1) + F(fWV + 3 * a + 2, p) * Wel(b, 2);
          return u - s;
        });
        if (tid == 0) {  // Cholesky of the 12 x 12 system (oracle_ba.cpp cholesky_solve, one block)
          double* A = S.S;
          for (int e = 0; e < 78; ++e) {
            int a = 0;
            while ((a + 1) * (a + 2) / 2 <= e) ++a;
            const int b = e - a * (a + 1) / 2;
            A[12 * a + b] = S.sums[e] + (a == b ? S.D2[a] : 0.0);
          }
          double* bb = S.rhs;
          for (int j = 0; j < 12; ++j) bb[j] = -S.g[j] + S.sums[78 + j];
          S.pd = chol_solve_small<12>(A, bb);
          if (S.pd)
            for (int j = 0; j < 12; ++j) S.delta[j] = bb[j];
        }
        __syncthreads();
        const bool pd = S.pd != 0;
        double model_cost_change = 0.0;
        if (pd) {
          // back substitution delta_p = V^-1 (-g_p - W^T delta_B) and the model cost change 1/2 delta^T (D^2 delta - g)
          double acc = 0.0;
          for (uint32_t p = tid; p < N; p += kBThreads) {
            double t3[3] = {-F(fG, p), -F(fG + 1, p), -F(fG + 2, p)};
            for (int v = 0; v < 2; ++v) {
              double m[2] = {0, 0};
              for (int a = 0; a < 2; ++a)
                for (int k = 0; k < 6; ++k) m[a] += F(fJc + 12 * v + 6 * a + k, p) * S.delta[6 * v + k];
              for (int k = 0; k < 3; ++k) t3[k] -= F(fJp + 6 * v + k, p) * m[0] + F(fJp + 6 * v + 3 + k, p) * m[1];
            }
            for (int i = 0; i < 3; ++i) {
              const double d = F(fVi + 3 * i, p) * t3[0] + F(fVi + 3 * i + 1, p) * t3[1] + F(fVi + 3 * i + 2, p) * t3[2];
              F(fDel + i, p) = d;
              acc += d * ((fmin(fmax(F(fD + i, p), 1e-6), 1e32) / lm.radius) * d - F(fG + i, p));
            }
          }
          acc = block_sum_fixed<kBThreads>(acc, S.red);
          double cam = 0.0;
          for (int j = 0; j < 12; ++j) cam += S.delta[j] * (S.D2[j] * S.delta[j] - S.g[j]);
          model_cost_change = 0.5 * (cam + acc);
        }
        bool accepted = false;
        if (lm.step_usable(pd, model_cost_change)) {
          // trial point and the parameter tolerance on the unscaled step
          double dn = 0.0, xn = 0.0;
          for (uint32_t p = tid; p < N; p += kBThreads)
            for (int i = 0; i < 3; ++i) {
              const double d = F(fDel + i, p) * F(fS + i, p), x = F(fX + 3 * cur + i, p);
              F(fX + 3 * (cur ^ 1) + i, p) = x + d;
              dn += d * d;
              xn += x * x;
            }
          dn = block_sum_fixed<kBThreads>(dn, S.red);
          xn = block_sum_fixed<kBThreads>(xn, S.red);
          for (int j = 0; j < 12; ++j) {
            const double d = S.delta[j] * S.scale[j];
            dn += d * d;
            xn += S.pose[j] * S.pose[j];
          }
          if (tid < 12) S.pose_new[tid] = S.pose[tid] + S.delta[tid] * S.scale[tid];
          __syncthreads();
          if (lm.step_too_small(dn, xn)) break;
          const double new_cost = total_cost(S.pose_new, cur ^ 1);
          if ((accepted = lm.accept(cost, new_cost, model_cost_change))) {
            cur ^= 1;
            __syncthreads();
            if (tid < 12) S.pose[tid] = S.pose_new[tid];
            cost = new_cost;
            __syncthreads();
            evaluate(false);
            if (lm.converged(grad_max())) break;
          }
        }
        if (!accepted && lm.reject()) break;
        __syncthreads();
      }
    __syncthreads();
    if (tid < 12) io[pid].pose[tid] = S.pose[tid];
    if (tid == 0) {
      io[pid].iterations = lm.iterations;
      io[pid].successful = lm.successful;
      io[pid].termination = lm.termination;
      io[pid].initial_cost = initial_cost;
      io[pid].final_cost = cost;
    }
  }
#undef F
}

// pairs [p0, p1) of the map on worker w
int relpose_range(r3d_ctx* ctx, DeviceWorker& w, const r3d_matches* m, const r3d_view_info* views, uint32_t n_views,
                  const r3d_relpose_options& opt, uint64_t p0, uint64_t p1, r3d_relative_pose* out,
                  std::vector<std::vector<r3d_indmatch>>& inl, r3d_relpose_timing& T) {
  const double t0 = now_ms();
  T = r3d_relpose_timing{};
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  for (uint64_t p = p0; p < p1; ++p) {
    r3d_relative_pose& o = out[p];
    std::memset(&o, 0, sizeof(o));
    o.I = m->pairs[2 * p];
    o.J = m->pairs[2 * p + 1];
    o.ba_termination = -1;
    if (o.I >= n_views || o.J >= n_views) return fail(ctx, R3D_ERR_INVALID, "r3d_relative_poses: view id outside views[]");
    o.status = m->per[p].size() <= 5 ? R3D_RELPOSE_TOO_FEW
               : (!(views[o.I].focal > 0.0) || !(views[o.J].focal > 0.0)) ? R3D_RELPOSE_NO_INTRINSIC
                                                                           : R3D_RELPOSE_NO_MODEL;
  }
  // ---- 1. robustRelativePose's AC-RANSAC (the essential filter's kernel) ----
  std::vector<AcBestModel> best(m->pairs.size() / 2);
  r3d_filter_timing FT{};
  {
    const int rc = filter_pairs_model(ctx, w, 2, opt.precision_px, opt.max_iter, m, views, n_views, p0, p1, FT, inl, &best);
    if (rc) return rc;
  }
  T.ms_ransac = FT.ms_device_total;
  T.kernel_launches += FT.kernel_launches;
  std::vector<uint64_t> cand;
  for (uint64_t p = p0; p < p1; ++p)
    if (out[p].status == R3D_RELPOSE_NO_MODEL && !inl[p].empty()) cand.push_back(p);
  if (cand.empty()) {
    T.ms_host = now_ms() - t0 - T.ms_ransac;
    return R3D_OK;
  }
  // ---- positions: the inliers (cheirality) and every match (bundle adjustment), promoted to double ----
  std::vector<RpPair> hp(cand.size());
  uint64_t n_in = 0, n_all = 0;
  for (size_t a = 0; a < cand.size(); ++a) {
    const uint64_t p = cand[a];
    r3d_relative_pose& o = out[p];
    RpPair& q = hp[a];
    q.in_ofs = (uint32_t)n_in; q.n_in = (uint32_t)inl[p].size();
    q.all_ofs = (uint32_t)n_all; q.M = (uint32_t)m->per[p].size();
    n_in += q.n_in;
    n_all += q.M;
    const r3d_view_info& vi = views[o.I];
    const r3d_view_info& vj = views[o.J];
    q.K[0] = vi.focal; q.K[1] = vi.ppx; q.K[2] = vi.ppy; q.K[3] = vj.focal; q.K[4] = vj.ppx; q.K[5] = vj.ppy;
    std::memcpy(q.F, best[p].model, sizeof(q.F));
    o.n_inliers = q.n_in;
    o.found_residual_precision = sqrt(best[p].errorMax);
  }
  if (n_all > 0xfffffff0ull) return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_relative_poses: too many matches in one call");
  std::vector<double2> hx1(n_in), hx2(n_in), ha1(opt.refine ? n_all : 0), ha2(opt.refine ? n_all : 0);
  parallel_for(ctx->host_threads, cand.size(), [&](size_t a) {
    const uint64_t p = cand[a];
    const std::vector<float>& xi = w.views.find(out[p].I)->second.h_xy;
    const std::vector<float>& xj = w.views.find(out[p].J)->second.h_xy;
    auto put = [&](const auto& v, double2* d1, double2* d2) {
      for (size_t k = 0; k < v.size(); ++k) {
        d1[k] = make_double2((double)xi[2 * (size_t)v[k].i], (double)xi[2 * (size_t)v[k].i + 1]);
        d2[k] = make_double2((double)xj[2 * (size_t)v[k].j], (double)xj[2 * (size_t)v[k].j + 1]);
      }
    };
    put(inl[p], &hx1[hp[a].in_ofs], &hx2[hp[a].in_ofs]);
    if (opt.refine) put(m->per[p], &ha1[hp[a].all_ofs], &ha2[hp[a].all_ofs]);  // indices checked by the filter's upload
  });
  const uint32_t nc = (uint32_t)cand.size();
  DevArr<RpPair> d_pairs(w);
  DevArr<double2> d_x1(w), d_x2(w), d_a1(w), d_a2(w);
  DevArr<RpCheir> d_ch(w);
  if (!d_pairs.alloc(nc) || !d_x1.alloc(n_in) || !d_x2.alloc(n_in) || !d_ch.alloc(nc))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_relative_poses: device scratch");
  Events<4> ev;
  R3D_CUDA_TRY(ctx, ev.create());
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_pairs.p, hp.data(), nc * sizeof(RpPair), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_x1.p, hx1.data(), n_in * sizeof(double2), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_x2.p, hx2.data(), n_in * sizeof(double2), cudaMemcpyHostToDevice, w.stream));
  // ---- 2. cheirality ----
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[0], w.stream));
  k_relpose_cheirality<<<nc, kCThreads, 0, w.stream>>>(d_pairs.p, d_x1.p, d_x2.p, d_ch.p);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[1], w.stream));
  T.kernel_launches += 1;
  std::vector<RpCheir> hch(nc);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hch.data(), d_ch.p, nc * sizeof(RpCheir), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  T.ms_cheirality = ev.ms(0, 1);
  std::vector<uint32_t> ok;  // candidates with a motion
  for (uint32_t a = 0; a < nc; ++a) {
    r3d_relative_pose& o = out[cand[a]];
    const RpCheir& c = hch[a];
    std::memcpy(o.E, c.E, sizeof(o.E));
    if (c.cnt[c.best] == 0) {
      o.status = R3D_RELPOSE_CHEIRALITY;
      continue;
    }
    o.status = R3D_RELPOSE_OK;
    std::memcpy(o.rotation, c.R, sizeof(o.rotation));
    std::memcpy(o.translation, c.t, sizeof(o.translation));
    ok.push_back(a);
  }
  // ---- 3. two-view bundle adjustment ----
  if (opt.refine && !ok.empty()) {
    std::vector<RpBa> hba(nc);
    uint32_t cap = 1;
    for (uint32_t a : ok) {
      RpBa& b = hba[a];
      std::memset(&b, 0, sizeof(b));
      std::memcpy(b.R, hch[a].R, sizeof(b.R));
      std::memcpy(b.t, hch[a].t, sizeof(b.t));
      rp::rotation_to_angle_axis(hch[a].R, b.pose + 6);
      for (int i = 0; i < 3; ++i) b.pose[9 + i] = hch[a].t[i];
      cap = std::max(cap, hp[a].M);
    }
    std::vector<uint32_t> order(ok);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return hp[x].M > hp[y].M; });
    // grid: one CTA per SM (the kernel needs ~170 registers per thread), fewer when the per-CTA scratch slots would pass
    // 4 GB
    const size_t slot = (size_t)kFields * cap * sizeof(double);
    uint32_t grid = std::min<uint32_t>((uint32_t)order.size(), (uint32_t)w.sm_count);
    grid = (uint32_t)std::max<size_t>(1, std::min<size_t>(grid, ((size_t)4 << 30) / slot));
    DevArr<RpBa> d_ba(w);
    DevArr<uint32_t> d_order(w), d_work(w);
    DevArr<double> d_scr(w);
    if (!d_a1.alloc(n_all) || !d_a2.alloc(n_all) || !d_ba.alloc(nc) || !d_order.alloc(order.size()) || !d_work.alloc(1) ||
        !d_scr.alloc(slot / sizeof(double) * grid))
      return fail(ctx, R3D_ERR_NOMEM, "r3d_relative_poses: device scratch");
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_a1.p, ha1.data(), n_all * sizeof(double2), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_a2.p, ha2.data(), n_all * sizeof(double2), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_ba.p, hba.data(), nc * sizeof(RpBa), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_order.p, order.data(), order.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_work.p, 0, sizeof(uint32_t), w.stream));
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[2], w.stream));
    k_relpose_ba<<<grid, kBThreads, 0, w.stream>>>(d_pairs.p, d_order.p, (uint32_t)order.size(), d_work.p, d_a1.p, d_a2.p, d_ba.p, lm_params(opt.ba),
                                                   d_scr.p, cap);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[3], w.stream));
    T.kernel_launches += 1;
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hba.data(), d_ba.p, nc * sizeof(RpBa), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    T.ms_refine = ev.ms(2, 3);
    for (uint32_t a : ok) {
      r3d_relative_pose& o = out[cand[a]];
      const RpBa& b = hba[a];
      o.ba_iterations = b.iterations;
      o.ba_successful_steps = b.successful;
      o.ba_termination = b.termination;
      o.ba_initial_cost = b.initial_cost;
      o.ba_final_cost = b.final_cost;
      T.ba_iterations += b.iterations;
      if (b.termination == 4) continue;  // Adjust() returned false: the unrefined motion stays
      // RelativeCameraMotion(R_I, t_I, R_J, t_J): R = R_J R_I^T, t = t_J - R t_I
      double RI[9], RJ[9], RIt[9];
      rp::angle_axis_to_rotation(b.pose, RI);
      rp::angle_axis_to_rotation(b.pose + 6, RJ);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) RIt[3 * r + c] = RI[3 * c + r];
      rp::matmul3(RJ, RIt, o.rotation);
      for (int i = 0; i < 3; ++i)
        o.translation[i] = b.pose[9 + i] - (o.rotation[3 * i] * b.pose[3] + o.rotation[3 * i + 1] * b.pose[4] + o.rotation[3 * i + 2] * b.pose[5]);
    }
  }
  T.ms_device_total = T.ms_ransac + T.ms_cheirality + T.ms_refine;
  T.ms_host = now_ms() - t0 - T.ms_device_total;
  return R3D_OK;
}

}  // namespace

}  // namespace r3d

using namespace r3d;

extern "C" void r3d_relpose_default_options(r3d_relpose_options* o) {
  if (!o) return;
  o->precision_px = 2.5;  // RelativePose_Info::initial_residual_tolerance = Square(2.5)
  o->max_iter = 256;      // robustRelativePose's ACRANSAC budget
  o->refine = 1;          // bRefine_using_BA = true
  r3d_ba_default_options(&o->ba);
  o->ba.refine_intrinsics = 0;  // Optimize_Options(Intrinsic_Parameter_Type::NONE, ADJUST_ALL, ADJUST_ALL)
}

extern "C" int r3d_relative_poses(r3d_ctx* ctx, const r3d_matches* matches, const r3d_view_info* views, uint32_t n_views,
                                  const r3d_relpose_options* opt, r3d_relative_pose* out, r3d_matches** inliers) {
  if (!ctx || !matches || !views || !opt || (!out && matches->pairs.size())) return fail(ctx, R3D_ERR_INVALID, "r3d_relative_poses: bad arguments");
  if (inliers) *inliers = nullptr;
  if (!(opt->precision_px > 0.0) || opt->max_iter == 0) return fail(ctx, R3D_ERR_INVALID, "r3d_relative_poses: bad AC-RANSAC options");
  if (opt->refine && opt->ba.refine_intrinsics)
    return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_relative_poses: the two-view refinement keeps the intrinsics fixed");
  const uint64_t P = matches->pairs.size() / 2;
  std::vector<std::vector<r3d_indmatch>> inl(P);
  // the pairs are independent: contiguous ranges of equal match counts, one per device (the rule of r3d_filter_pairs)
  const std::vector<uint64_t> cut = balanced_cuts(P, ctx->workers.size(), [&](uint64_t p) { return matches->per[p].size(); });
  std::vector<r3d_relpose_timing> tms(ctx->workers.size());
  const int rc = fan_out(ctx, [&](size_t k, DeviceWorker& w) {
    return relpose_range(ctx, w, matches, views, n_views, *opt, cut[k], cut[k + 1], out, inl, tms[k]);
  });
  if (rc) return rc;
  r3d_relpose_timing sum{};
  for (const r3d_relpose_timing& t : tms) {
    sum.ms_ransac = std::max(sum.ms_ransac, t.ms_ransac);
    sum.ms_cheirality = std::max(sum.ms_cheirality, t.ms_cheirality);
    sum.ms_refine = std::max(sum.ms_refine, t.ms_refine);
    sum.ms_device_total = std::max(sum.ms_device_total, t.ms_device_total);
    sum.ms_host = std::max(sum.ms_host, t.ms_host);
    sum.kernel_launches += t.kernel_launches;
    sum.ba_iterations += t.ba_iterations;
  }
  ctx->relpose_timing = sum;
  if (inliers) {
    r3d_matches* mm = new r3d_matches();
    for (uint64_t p = 0; p < P; ++p)
      if (out[p].status == R3D_RELPOSE_OK) mm->push(matches->pairs[2 * p], matches->pairs[2 * p + 1], std::move(inl[p]));
    *inliers = mm;
  }
  return R3D_OK;
}

extern "C" int r3d_get_relpose_timing(const r3d_ctx* ctx, r3d_relpose_timing* out) {
  if (!ctx || !out) return R3D_ERR_INVALID;
  *out = ctx->relpose_timing;
  return R3D_OK;
}
