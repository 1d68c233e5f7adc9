/*
 * oracle_resection.h -- C ABI of the CPU ORACLE of the resection step (liboracle_resection.so, oracle/resection.mk).
 * TEST INFRASTRUCTURE ONLY, like oracle.h: the residual Jacobians it calls are liboracle.so's own orc_ba_jacobian_model.
 */
#ifndef R3D_ORACLE_RESECTION_H
#define R3D_ORACLE_RESECTION_H
#include "oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- absolute pose of a view from 2D-3D correspondences (SfM_Localizer::Localize + RefinePose) ---- */
#define ORC_RESECT_OK 0
#define ORC_RESECT_TOO_FEW 1
#define ORC_RESECT_NO_INTRINSIC 2
#define ORC_RESECT_NO_MODEL 3
typedef struct {
  double precision_px;         /* +inf: pure a-contrario */
  uint32_t max_iter;           /* 4096 */
  int refine;                  /* RefinePose: pose only */
  orc_ba_options ba;           /* refine_intrinsics must be 0 */
} orc_resection_options;
/* same layout as r3d_resection (include/r3dgpu.h) */
typedef struct {
  uint32_t view_id;
  int status;
  uint32_t n_inliers;
  double found_residual_precision;
  double rotation[9], center[3], translation[3];
  double rotation_ransac[9], translation_ransac[3];
  uint32_t lm_iterations, lm_successful_steps;
  int lm_termination;          /* -1: not refined */
  double lm_initial_cost, lm_final_cost;
} orc_resection_result;

/* camera parameters everywhere below: intr8 = f, ppx, ppy, then the model's distortion coefficients (K1: k1 | K3: k1 k2
 * k3 | Brown T2: k1 k2 k3 t1 t2 | fisheye: k1 k2 k3 k4), model = openMVG EINTRINSIC 1..5 */
/* P3P: K = f, ppx, ppy; X 3 x 3 world points; x 3 x 2 undistorted pixels; P: up to 4 models K [R | t], 3 x 4 row-major */
int orc_p3p(const double* K, const double* X, const double* x, double* P /* 48 */);
/* get_ud_pixel by a fixed number of Newton steps: xy, out n x 2 */
void orc_undistort(int model, const double* intr8, const double* xy, uint32_t n, double* out);
/* pose-only Levenberg-Marquardt from pose (angle-axis | t, in/out) over N correspondences; returns s->termination */
int orc_resect_refine(int model, const double* intr8, const double* X, const double* x, uint32_t N, const orc_ba_options* o,
                      double* pose, orc_ba_summary* s);
/* one view: X M x 3, x M x 2 (original pixels); inliers (capacity M): AC-RANSAC inliers in residual order.  Returns
 * r->status. */
int orc_resect_view(const double* X, const double* x, uint32_t M, uint32_t width, uint32_t height, int model,
                    const double* intr8, const orc_resection_options* o, orc_resection_result* r, uint32_t* inliers);
/* a batch (omp over views); first / count: each view's correspondences in X / x; inl (capacity = all correspondences)
 * and inl_ofs (n + 1): the inliers of every view */
void orc_resect_views(uint32_t n, const uint64_t* first, const uint64_t* count, const uint32_t* widths, const uint32_t* heights,
                      const int* models, const double* intr8, const double* X, const double* x, const orc_resection_options* o,
                      orc_resection_result* out, uint32_t* inl, uint64_t* inl_ofs, int n_threads);

#ifdef __cplusplus
}
#endif
#endif
