// oracle_relpose.cpp -- CPU ORACLE (test infrastructure; see oracle_relpose.h).
//
// Restates the loop body of GlobalSfMReconstructionEngine_RelativeMotions::Compute_Relative_Rotations, the first
// step of the global pipeline the reference drives on matches.e.txt (src/threads/R3DTriangulationThread.cpp:201-250;
// un-vendored OpenMVG 1.4 sfm_global_engine_relative_motions.cpp + sfm_robust_model_estimation.cpp, SURVEY.md A.9):
//   * robustRelativePose: ACRANSAC with the essential adaptor (orc_acransac_E: the E filter's state machine and RNG
//     stream), initial_residual_tolerance = Square(2.5), 256 iterations; rejected when minNFA >= 0 or
//     #inliers < 2.5 * 5;
//   * MotionFromEssential + the cheirality test: the four motions of E, every inlier triangulated by DLT from its
//     bearing vectors, the first motion with the most points in front of both cameras (none: rejected);
//   * bRefine_using_BA: the two-view scene (pose I = (I, 0), pose J = the motion, EVERY match of the pair
//     triangulated by DLT in pixels with P = K [R | t]) refined by Bundle_Adjustment_Ceres (poses + structure,
//     intrinsics fixed, Huber(Square(4))); on success R_rel = R_J R_I^T, t_rel = t_J - R_rel t_I, on failure the
//     unrefined motion is kept.
// Deliberate, documented deviations (DESIGN.md sec. 2):
//   * E = K2^T F K1 from the F of the best model that orc_acransac_E reports (F = K2^-T E K1^-1 of the 5-point
//     solver's E): the solver's E up to rounding and with the same scale;
//   * Eigen::JacobiSVD of E -> cyclic one-sided Jacobi with a fixed number of sweeps (basic operations only; the
//     device restates it, relpose_math.cuh); U's third column is u0 x u1;
//   * TriangulateDLT (SVD null vector of the 4x4 system) -> the inhomogeneous DLT: 3x3 normal equations, adjugate
//     inverse (the oracle's triangulation, oracle_sfm.cpp);
//   * the R -> angle-axis conversion is Ceres' RotationMatrixToAngleAxis (quaternion path).
// PARITY UNPINNED.
#include "oracle_relpose.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include <omp.h>

namespace orc {
namespace rp {

constexpr int kSvdSweeps = 8;

// A = U diag(S) V^T for a 3x3 A (row-major), S descending; one-sided Jacobi on the columns of A, fixed sweep count.
// U's third column is u0 x u1 (E has rank 2, its own third column carries no direction).
void svd3(const double* A, double* U, double* S, double* V) {
  double B[9], Vm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) B[i] = A[i];
  for (int sweep = 0; sweep < kSvdSweeps; ++sweep)
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double alpha = 0.0, beta = 0.0, gamma = 0.0;
      for (int i = 0; i < 3; ++i) {
        alpha = alpha + B[3 * i + p] * B[3 * i + p];
        beta = beta + B[3 * i + q] * B[3 * i + q];
        gamma = gamma + B[3 * i + p] * B[3 * i + q];
      }
      if (gamma == 0.0) continue;
      const double zeta = (beta - alpha) / (2.0 * gamma);
      const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
      for (int i = 0; i < 3; ++i) {
        const double bp = B[3 * i + p], bq = B[3 * i + q];
        B[3 * i + p] = c * bp - s * bq;
        B[3 * i + q] = s * bp + c * bq;
        const double vp = Vm[3 * i + p], vq = Vm[3 * i + q];
        Vm[3 * i + p] = c * vp - s * vq;
        Vm[3 * i + q] = s * vp + c * vq;
      }
    }
  double s[3];
  for (int k = 0; k < 3; ++k) s[k] = std::sqrt(B[k] * B[k] + B[3 + k] * B[3 + k] + B[6 + k] * B[6 + k]);
  int o[3] = {0, 1, 2};
  if (s[o[1]] > s[o[0]]) std::swap(o[0], o[1]);
  if (s[o[2]] > s[o[1]]) std::swap(o[1], o[2]);
  if (s[o[1]] > s[o[0]]) std::swap(o[0], o[1]);
  for (int k = 0; k < 3; ++k) {
    S[k] = s[o[k]];
    for (int i = 0; i < 3; ++i) V[3 * i + k] = Vm[3 * i + o[k]];
  }
  for (int k = 0; k < 2; ++k)
    for (int i = 0; i < 3; ++i) U[3 * i + k] = B[3 * i + o[k]] / S[k];
  U[2] = U[3] * U[7] - U[6] * U[4];
  U[5] = U[6] * U[1] - U[0] * U[7];
  U[8] = U[0] * U[4] - U[3] * U[1];
}

double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

void matmul3(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}

// E = K2^T F K1, K = [f 0 ppx; 0 f ppy; 0 0 1] (Kpair: f, ppx, ppy of I, then of J)
void essential_from_fundamental(const double* F, const double* K1, const double* K2, double* E) {
  const double k1[9] = {K1[0], 0.0, K1[1], 0.0, K1[0], K1[2], 0.0, 0.0, 1.0};
  const double k2[9] = {K2[0], 0.0, K2[1], 0.0, K2[0], K2[2], 0.0, 0.0, 1.0};
  double T[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double a = 0.0;
      for (int k = 0; k < 3; ++k) a = a + k2[3 * k + r] * F[3 * k + c];  // K2^T F
      T[3 * r + c] = a;
    }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double a = 0.0;
      for (int k = 0; k < 3; ++k) a = a + T[3 * r + k] * k1[3 * k + c];
      E[3 * r + c] = a;
    }
}

// MotionFromEssential (multiview/solver_essential_kernel.cpp): Rs = {UWV^T, UWV^T, UW^TV^T, UW^TV^T},
// ts = {u2, -u2, u2, -u2}
void motions_from_essential(const double* E, double* Rs, double* ts) {
  double U[9], S[3], V[9];
  svd3(E, U, S, V);
  if (det3(U) < 0.0)
    for (int i = 0; i < 3; ++i) U[3 * i + 2] = -U[3 * i + 2];
  double Vt[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Vt[3 * r + c] = V[3 * c + r];
  if (det3(Vt) < 0.0)
    for (int c = 0; c < 3; ++c) Vt[6 + c] = -Vt[6 + c];
  const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
  double T[9], R1[9], R2[9];
  matmul3(U, W, T);
  matmul3(T, Vt, R1);
  matmul3(U, Wt, T);
  matmul3(T, Vt, R2);
  for (int k = 0; k < 4; ++k) {
    std::memcpy(Rs + 9 * k, k < 2 ? R1 : R2, 9 * sizeof(double));
    const double sg = (k & 1) ? -1.0 : 1.0;
    for (int i = 0; i < 3; ++i) ts[3 * k + i] = sg * U[3 * i + 2];
  }
}

// inhomogeneous two-view DLT: rows x0 P.row2 - x2 P.row0, x1 P.row2 - x2 P.row1 of both views (P 3x4 row-major,
// x homogeneous), normal equations solved by the adjugate
void triangulate2(const double* P1, const double* x1, const double* P2, const double* x2, double* X) {
  double r[4][4];
  const double* Ps[2] = {P1, P2};
  const double* xs[2] = {x1, x2};
  for (int v = 0; v < 2; ++v)
    for (int j = 0; j < 4; ++j) {
      r[2 * v][j] = xs[v][0] * Ps[v][8 + j] - xs[v][2] * Ps[v][j];
      r[2 * v + 1][j] = xs[v][1] * Ps[v][8 + j] - xs[v][2] * Ps[v][4 + j];
    }
  double a[9], b[3];
  for (int k = 0; k < 3; ++k) {
    for (int j = 0; j < 3; ++j) a[3 * k + j] = ((r[0][k] * r[0][j] + r[1][k] * r[1][j]) + r[2][k] * r[2][j]) + r[3][k] * r[3][j];
    b[k] = -(((r[0][k] * r[0][3] + r[1][k] * r[1][3]) + r[2][k] * r[2][3]) + r[3][k] * r[3][3]);
  }
  const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
  const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
  const double inv[9] = {c00 / det, (a[2] * a[7] - a[1] * a[8]) / det, (a[1] * a[5] - a[2] * a[4]) / det,
                         c01 / det, (a[0] * a[8] - a[2] * a[6]) / det, (a[2] * a[3] - a[0] * a[5]) / det,
                         c02 / det, (a[1] * a[6] - a[0] * a[7]) / det, (a[0] * a[4] - a[1] * a[3]) / det};
  for (int i = 0; i < 3; ++i) X[i] = inv[3 * i] * b[0] + inv[3 * i + 1] * b[1] + inv[3 * i + 2] * b[2];
}

// [R | t] (3x4 row-major) of a motion
void rt_matrix(const double* R, const double* t, double* P) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) P[4 * i + j] = R[3 * i + j];
    P[4 * i + 3] = t[i];
  }
}

// cheirality point of one inlier under one motion: in front of both cameras
bool in_front(const double* P2, const double* b1, const double* b2) {
  const double P1[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  double X[3];
  triangulate2(P1, b1, P2, b2, X);
  const double z2 = P2[8] * X[0] + P2[9] * X[1] + P2[10] * X[2] + P2[11];
  return X[2] > 0.0 && z2 > 0.0;
}

// bearing vector (Pinhole_Intrinsic::operator(), as oracle_acransac.cpp)
void bearing(const double* K, double x, double y, double* b) {
  const double kinv00 = 1.0 / K[0], kinv02 = -K[1] / K[0], kinv12 = -K[2] / K[0];
  const double bx = kinv00 * x + kinv02, by = kinv00 * y + kinv12, bz = 1.0;
  const double n = std::sqrt((bx * bx + by * by) + bz * bz);
  b[0] = bx / n; b[1] = by / n; b[2] = bz / n;
}

// get_projective_equivalent: K [R | t]
void projective(const double* K, const double* R, const double* t, double* P) {
  for (int j = 0; j < 3; ++j) {
    P[j] = K[0] * R[j] + K[1] * R[6 + j];
    P[4 + j] = K[0] * R[3 + j] + K[2] * R[6 + j];
    P[8 + j] = R[6 + j];
  }
  P[3] = K[0] * t[0] + K[1] * t[2];
  P[7] = K[0] * t[1] + K[2] * t[2];
  P[11] = t[2];
}

// ceres::RotationMatrixToAngleAxis (RotationMatrixToQuaternion + QuaternionToAngleAxis), R row-major
void rotation_to_angle_axis(const double* R, double* aa) {
  double q[4];
  const double trace = R[0] + R[4] + R[8];
  if (trace >= 0.0) {
    double t = std::sqrt(trace + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (R[7] - R[5]) * t;
    q[2] = (R[2] - R[6]) * t;
    q[3] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = std::sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i + 1] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (R[3 * k + j] - R[3 * j + k]) * t;
    q[j + 1] = (R[3 * j + i] + R[3 * i + j]) * t;
    q[k + 1] = (R[3 * k + i] + R[3 * i + k]) * t;
  }
  const double s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  double k = 2.0;
  if (s2 > 0.0) {
    const double st = std::sqrt(s2), ct = q[0];
    const double two_theta = 2.0 * (ct < 0.0 ? std::atan2(-st, -ct) : std::atan2(st, ct));
    k = two_theta / st;
  }
  for (int i = 0; i < 3; ++i) aa[i] = q[i + 1] * k;
}

// ceres::AngleAxisToRotationMatrix, R row-major
void angle_axis_to_rotation(const double* aa, double* R) {
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > 2.220446049250313e-16) {
    const double th = std::sqrt(th2);
    const double wx = aa[0] / th, wy = aa[1] / th, wz = aa[2] / th;
    const double c = std::cos(th), s = std::sin(th), oc = 1.0 - c;
    R[0] = c + wx * wx * oc;      R[1] = wx * wy * oc - wz * s; R[2] = wy * s + wx * wz * oc;
    R[3] = wz * s + wx * wy * oc; R[4] = c + wy * wy * oc;      R[5] = -wx * s + wy * wz * oc;
    R[6] = -wy * s + wx * wz * oc; R[7] = wx * s + wy * wz * oc; R[8] = c + wz * wz * oc;
  } else {
    R[0] = 1.0;    R[1] = -aa[2]; R[2] = aa[1];
    R[3] = aa[2];  R[4] = 1.0;    R[5] = -aa[0];
    R[6] = -aa[1]; R[7] = aa[0];  R[8] = 1.0;
  }
}

}  // namespace rp
}  // namespace orc

using namespace orc::rp;

extern "C" {

void orc_motions_from_essential(const double* E, double* Rs, double* ts) { motions_from_essential(E, Rs, ts); }

int orc_relative_pose(const double* xI, const double* xJ, uint32_t M, uint32_t wI, uint32_t hI, uint32_t wJ, uint32_t hJ,
                      const double* Kpair, const orc_relpose_options* o, orc_relpose_result* r, uint32_t* inliers) {
  const uint32_t I = r->I, J = r->J;
  std::memset(r, 0, sizeof(*r));
  r->I = I;
  r->J = J;
  r->ba_termination = -1;
  if (M <= 5) return r->status = ORC_RELPOSE_TOO_FEW;
  if (!(Kpair[0] > 0.0) || !(Kpair[3] > 0.0)) return r->status = ORC_RELPOSE_NO_INTRINSIC;
  std::vector<uint32_t> inl(M);
  double info[3], F[9];
  // keeps the pair iff minNFA < 0 and #inliers > 2.5 * 5, i.e. returns 0 in every other case
  const int64_t n = orc_acransac_E(xI, xJ, M, wI, hI, wJ, hJ, Kpair, o->precision_px, o->max_iter, inl.data(), F, info);
  if (n == 0) return r->status = ORC_RELPOSE_NO_MODEL;
  inl.resize((size_t)n);
  essential_from_fundamental(F, Kpair, Kpair + 3, r->E);
  r->n_inliers = (uint32_t)n;
  r->found_residual_precision = info[1];
  std::memcpy(inliers, inl.data(), inl.size() * sizeof(uint32_t));
  // ---- cheirality: the first motion with the most inliers in front of both cameras ----
  double Rs[36], ts[12], P2[4][12];
  motions_from_essential(r->E, Rs, ts);
  for (int k = 0; k < 4; ++k) rt_matrix(Rs + 9 * k, ts + 3 * k, P2[k]);
  uint32_t cnt[4] = {0, 0, 0, 0};
  for (uint32_t idx : inl) {
    double b1[3], b2[3];
    bearing(Kpair, xI[2 * idx], xI[2 * idx + 1], b1);
    bearing(Kpair + 3, xJ[2 * idx], xJ[2 * idx + 1], b2);
    for (int k = 0; k < 4; ++k) cnt[k] += in_front(P2[k], b1, b2) ? 1u : 0u;
  }
  int best = 0;
  for (int k = 1; k < 4; ++k)
    if (cnt[k] > cnt[best]) best = k;
  if (cnt[best] == 0) return r->status = ORC_RELPOSE_CHEIRALITY;
  std::memcpy(r->rotation, Rs + 9 * best, 9 * sizeof(double));
  std::memcpy(r->translation, ts + 3 * best, 3 * sizeof(double));
  r->status = ORC_RELPOSE_OK;
  if (!o->refine) return r->status;
  // ---- two-view bundle adjustment over every match of the pair ----
  const double Id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, zero[3] = {0, 0, 0};
  double PI[12], PJ[12];
  projective(Kpair, Id, zero, PI);
  projective(Kpair + 3, r->rotation, r->translation, PJ);
  std::vector<double> poses(12, 0.0), intr(12, 0.0), pts(3 * (size_t)M), obs_xy(4 * (size_t)M);
  std::vector<uint32_t> obs_cam(2 * (size_t)M), obs_pt(2 * (size_t)M);
  rotation_to_angle_axis(r->rotation, &poses[6]);
  for (int i = 0; i < 3; ++i) poses[9 + i] = r->translation[i];
  for (int g = 0; g < 2; ++g)
    for (int i = 0; i < 3; ++i) intr[6 * g + i] = Kpair[3 * g + i];
  for (uint32_t k = 0; k < M; ++k) {
    const double h1[3] = {xI[2 * k], xI[2 * k + 1], 1.0}, h2[3] = {xJ[2 * k], xJ[2 * k + 1], 1.0};
    triangulate2(PI, h1, PJ, h2, &pts[3 * (size_t)k]);
    obs_cam[2 * k] = 0; obs_cam[2 * k + 1] = 1;
    obs_pt[2 * k] = k; obs_pt[2 * k + 1] = k;
    obs_xy[4 * (size_t)k] = xI[2 * k]; obs_xy[4 * (size_t)k + 1] = xI[2 * k + 1];
    obs_xy[4 * (size_t)k + 2] = xJ[2 * k]; obs_xy[4 * (size_t)k + 3] = xJ[2 * k + 1];
  }
  const uint32_t cam_intr[2] = {0, 1};
  orc_ba_problem p;
  std::memset(&p, 0, sizeof(p));
  p.n_cams = 2; p.n_pts = M; p.n_intr = 2; p.n_obs = 2 * (uint64_t)M;
  p.poses = poses.data(); p.intrinsics = intr.data(); p.points = pts.data();
  p.obs_cam = obs_cam.data(); p.obs_pt = obs_pt.data(); p.cam_intr = cam_intr; p.obs_xy = obs_xy.data();
  orc_ba_options bo = o->ba;
  bo.refine_intrinsics = 0;
  bo.n_threads = 1;
  orc_ba_summary s;
  orc_bundle_adjust(&p, &bo, &s, nullptr);
  r->ba_iterations = s.iterations;
  r->ba_successful_steps = s.successful_steps;
  r->ba_termination = s.termination;
  r->ba_initial_cost = s.initial_cost;
  r->ba_final_cost = s.final_cost;
  if (s.termination == 4) return r->status;  // Adjust() returned false: the unrefined motion stays
  // RelativeCameraMotion(R_I, t_I, R_J, t_J)
  double RI[9], RJ[9];
  angle_axis_to_rotation(&poses[0], RI);
  angle_axis_to_rotation(&poses[6], RJ);
  double RIt[9];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) RIt[3 * a + b] = RI[3 * b + a];
  matmul3(RJ, RIt, r->rotation);
  for (int i = 0; i < 3; ++i)
    r->translation[i] = poses[9 + i] - (r->rotation[3 * i] * poses[3] + r->rotation[3 * i + 1] * poses[4] + r->rotation[3 * i + 2] * poses[5]);
  return r->status;
}

int64_t orc_relative_poses(const float* const* xys, const uint32_t* widths, const uint32_t* heights, const double* Ks,
                           uint32_t n_views, const uint32_t* pairs, uint64_t P, const uint64_t* put_ofs, const orc_indmatch* put,
                           const orc_relpose_options* o, orc_relpose_result* out, uint64_t* inl_ofs, orc_indmatch* inl,
                           int n_threads) {
  (void)n_views;
  if (n_threads <= 0) n_threads = omp_get_max_threads();
  std::vector<std::vector<orc_indmatch>> res(P);
#pragma omp parallel for schedule(dynamic) num_threads(n_threads)
  for (int64_t p = 0; p < (int64_t)P; ++p) {
    const uint32_t I = pairs[2 * p], J = pairs[2 * p + 1];
    const uint64_t b = put_ofs[p];
    const uint32_t M = (uint32_t)(put_ofs[p + 1] - b);
    std::vector<double> xI(2 * (size_t)M), xJ(2 * (size_t)M);
    for (uint32_t k = 0; k < M; ++k) {
      xI[2 * k] = (double)xys[I][2 * (size_t)put[b + k].i];
      xI[2 * k + 1] = (double)xys[I][2 * (size_t)put[b + k].i + 1];
      xJ[2 * k] = (double)xys[J][2 * (size_t)put[b + k].j];
      xJ[2 * k + 1] = (double)xys[J][2 * (size_t)put[b + k].j + 1];
    }
    const double Kpair[6] = {Ks[3 * I], Ks[3 * I + 1], Ks[3 * I + 2], Ks[3 * J], Ks[3 * J + 1], Ks[3 * J + 2]};
    std::vector<uint32_t> idx(std::max<uint32_t>(M, 1));
    out[p].I = I;
    out[p].J = J;
    if (orc_relative_pose(xI.data(), xJ.data(), M, widths[I], heights[I], widths[J], heights[J], Kpair, o, &out[p], idx.data()) ==
        ORC_RELPOSE_OK)
      for (uint32_t k = 0; k < out[p].n_inliers; ++k) res[p].push_back(put[b + idx[k]]);
  }
  uint64_t ofs = 0;
  for (uint64_t p = 0; p < P; ++p) {
    inl_ofs[p] = ofs;
    std::memcpy(inl + ofs, res[p].data(), res[p].size() * sizeof(orc_indmatch));
    ofs += res[p].size();
  }
  inl_ofs[P] = ofs;
  return (int64_t)ofs;
}

}  // extern "C"
