// relpose_math.cuh -- the small dense steps of the relative-pose pipeline (relpose.cu), host + device.
// Every routine uses basic IEEE operations only (plus sqrt), so a translation unit compiled with --fmad=false computes
// exactly what the CPU restatement (oracle/oracle_relpose.cpp) computes; the discrete decisions taken from them (the
// cheirality counts, the chosen motion) are bit-identical.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define R3D_RP_HD __host__ __device__ __forceinline__
#else
#define R3D_RP_HD inline
#endif

namespace r3d {
namespace rp {

constexpr int kSvdSweeps = 8;

// A = U diag(S) V^T for a 3x3 A (row-major), S descending.  Replaces Eigen::JacobiSVD with cyclic one-sided Jacobi on
// the columns of A and a fixed sweep count (quadratic convergence: 8 sweeps are far more than a 3x3 needs).  U's third
// column is u0 x u1: an essential matrix has rank 2 and its third left singular vector is only defined up to sign.
R3D_RP_HD void svd3(const double* A, double* U, double* S, double* V) {
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
      const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
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
  for (int k = 0; k < 3; ++k) s[k] = sqrt(B[k] * B[k] + B[3 + k] * B[3 + k] + B[6 + k] * B[6 + k]);
  int o[3] = {0, 1, 2};
  int tmp;
  if (s[o[1]] > s[o[0]]) { tmp = o[0]; o[0] = o[1]; o[1] = tmp; }
  if (s[o[2]] > s[o[1]]) { tmp = o[1]; o[1] = o[2]; o[2] = tmp; }
  if (s[o[1]] > s[o[0]]) { tmp = o[0]; o[0] = o[1]; o[1] = tmp; }
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

R3D_RP_HD double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

R3D_RP_HD void matmul3(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}

// E = K2^T F K1, K = (f, ppx, ppy) -> [f 0 ppx; 0 f ppy; 0 0 1]: the essential matrix behind AC-RANSAC's model
// F = K2^-T E K1^-1 (the 5-point solver's E up to rounding, with its scale)
R3D_RP_HD void essential_from_fundamental(const double* F, const double* K1, const double* K2, double* E) {
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

// MotionFromEssential (OpenMVG multiview/solver_essential_kernel.cpp): U, V^T with positive determinant,
// Rs = {U W V^T, U W V^T, U W^T V^T, U W^T V^T} (row-major, 4 x 9), ts = {u2, -u2, u2, -u2}
R3D_RP_HD void motions_from_essential(const double* E, double* Rs, double* ts) {
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
    for (int i = 0; i < 9; ++i) Rs[9 * k + i] = k < 2 ? R1[i] : R2[i];
    const double sg = (k & 1) ? -1.0 : 1.0;
    for (int i = 0; i < 3; ++i) ts[3 * k + i] = sg * U[3 * i + 2];
  }
}

// Two-view DLT (replaces TriangulateDLT's SVD null vector): rows x0 P.row2 - x2 P.row0 and x1 P.row2 - x2 P.row1 of
// both views (P 3x4 row-major, x homogeneous), inhomogeneous least squares by the 3x3 normal equations + adjugate
R3D_RP_HD void triangulate2(const double* P1, const double* x1, const double* P2, const double* x2, double* X) {
  double r[4][4];
  for (int j = 0; j < 4; ++j) {
    r[0][j] = x1[0] * P1[8 + j] - x1[2] * P1[j];
    r[1][j] = x1[1] * P1[8 + j] - x1[2] * P1[4 + j];
    r[2][j] = x2[0] * P2[8 + j] - x2[2] * P2[j];
    r[3][j] = x2[1] * P2[8 + j] - x2[2] * P2[4 + j];
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

// [R | t] of a motion (3x4 row-major)
R3D_RP_HD void rt_matrix(const double* R, const double* t, double* P) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) P[4 * i + j] = R[3 * i + j];
    P[4 * i + 3] = t[i];
  }
}

// cheirality of one inlier under one motion [R | t]: Depth > 0 in camera I = [I | 0] and in camera J
R3D_RP_HD bool in_front(const double* P2, const double* b1, const double* b2) {
  const double P1[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  double X[3];
  triangulate2(P1, b1, P2, b2, X);
  const double z2 = P2[8] * X[0] + P2[9] * X[1] + P2[10] * X[2] + P2[11];
  return X[2] > 0.0 && z2 > 0.0;
}

// bearing vector of a pixel, (K^-1 [x y 1]^T).normalized() (Pinhole_Intrinsic::operator())
R3D_RP_HD void bearing_vec(const double* K, double x, double y, double* b) {
  const double kinv00 = 1.0 / K[0], kinv02 = -K[1] / K[0], kinv12 = -K[2] / K[0];
  const double bx = kinv00 * x + kinv02, by = kinv00 * y + kinv12, bz = 1.0;
  const double n = sqrt((bx * bx + by * by) + bz * bz);
  b[0] = bx / n; b[1] = by / n; b[2] = bz / n;
}

// get_projective_equivalent: K [R | t], K = (f, ppx, ppy)
R3D_RP_HD void projective(const double* K, const double* R, const double* t, double* P) {
  for (int j = 0; j < 3; ++j) {
    P[j] = K[0] * R[j] + K[1] * R[6 + j];
    P[4 + j] = K[0] * R[3 + j] + K[2] * R[6 + j];
    P[8 + j] = R[6 + j];
  }
  P[3] = K[0] * t[0] + K[1] * t[2];
  P[7] = K[0] * t[1] + K[2] * t[2];
  P[11] = t[2];
}

// ceres::RotationMatrixToAngleAxis (RotationMatrixToQuaternion + QuaternionToAngleAxis), R row-major.  The two-view
// BA's initial pose is converted on the host, where the oracle converts it, with the same libm; the pose refinement
// of resection.cu converts on the device, r3d_sfm::flatten (sfm_scene.cpp) the SfM_Data poses on the host.
R3D_RP_HD void rotation_to_angle_axis(const double* R, double* aa) {
  double q[4];
  const double trace = R[0] + R[4] + R[8];
  if (trace >= 0.0) {
    double t = sqrt(trace + 1.0);
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
    double t = sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i + 1] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (R[3 * k + j] - R[3 * j + k]) * t;
    q[j + 1] = (R[3 * j + i] + R[3 * i + j]) * t;
    q[k + 1] = (R[3 * k + i] + R[3 * i + k]) * t;
  }
  const double s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  double k = 2.0;
  if (s2 > 0.0) {
    const double st = sqrt(s2), ct = q[0];
    const double two_theta = 2.0 * (ct < 0.0 ? atan2(-st, -ct) : atan2(st, ct));
    k = two_theta / st;
  }
  for (int i = 0; i < 3; ++i) aa[i] = q[i + 1] * k;
}

// ceres::AngleAxisToRotationMatrix, R row-major (host)
inline void angle_axis_to_rotation(const double* aa, double* R) {
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > 2.220446049250313e-16) {
    const double th = sqrt(th2);
    const double wx = aa[0] / th, wy = aa[1] / th, wz = aa[2] / th;
    const double c = cos(th), s = sin(th), oc = 1.0 - c;
    R[0] = c + wx * wx * oc;       R[1] = wx * wy * oc - wz * s;  R[2] = wy * s + wx * wz * oc;
    R[3] = wz * s + wx * wy * oc;  R[4] = c + wy * wy * oc;       R[5] = -wx * s + wy * wz * oc;
    R[6] = -wy * s + wx * wz * oc; R[7] = wx * s + wy * wz * oc;  R[8] = c + wz * wz * oc;
  } else {
    R[0] = 1.0;    R[1] = -aa[2]; R[2] = aa[1];
    R[3] = aa[2];  R[4] = 1.0;    R[5] = -aa[0];
    R[6] = -aa[1]; R[7] = aa[0];  R[8] = 1.0;
  }
}

}  // namespace rp
}  // namespace r3d
