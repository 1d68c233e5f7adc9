/*
 * oracle_relpose.h -- C ABI of the CPU ORACLE of the relative-pose step (liboracle_relpose.so, oracle/relpose.mk).
 * TEST INFRASTRUCTURE ONLY, like oracle.h: the AC-RANSAC and bundle adjustment it calls are liboracle.so's own
 * orc_acransac_E and orc_bundle_adjust.
 */
#ifndef R3D_ORACLE_RELPOSE_H
#define R3D_ORACLE_RELPOSE_H
#include "oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- relative pose of an image pair (GlobalSfMReconstructionEngine_RelativeMotions::Compute_Relative_Rotations) ---- */
#define ORC_RELPOSE_OK 0
#define ORC_RELPOSE_TOO_FEW 1
#define ORC_RELPOSE_NO_INTRINSIC 2
#define ORC_RELPOSE_NO_MODEL 3
#define ORC_RELPOSE_CHEIRALITY 4
typedef struct {
  double precision_px;         /* 2.5 (initial_residual_tolerance = Square(2.5)) */
  uint32_t max_iter;           /* 256 */
  int refine;                  /* bRefine_using_BA: two-view BA of the pair */
  orc_ba_options ba;           /* refine_intrinsics must be 0 */
} orc_relpose_options;
/* same layout as r3d_relative_pose (include/r3dgpu.h) */
typedef struct {
  uint32_t I, J;
  int status;
  uint32_t n_inliers;
  double found_residual_precision;   /* ACRANSAC errorMax, px */
  double E[9];                       /* the 5-point solver's E of the best model */
  double rotation[9], translation[3];/* X_J = R X_I + t */
  uint32_t ba_iterations, ba_successful_steps;
  int ba_termination;                /* -1: not refined */
  double ba_initial_cost, ba_final_cost;
} orc_relpose_result;
/* MotionFromEssential with the fixed-sweep Jacobi SVD: Rs 4 x 9 (row-major), ts 4 x 3 */
void orc_motions_from_essential(const double* E, double* Rs, double* ts);
/* one pair: positions M x 2 (pixels), Kpair = f1 ppx1 ppy1 f2 ppx2 ppy2; inliers (capacity M): AC-RANSAC inliers in
 * residual order (n_inliers of them).  Returns r->status. */
int orc_relative_pose(const double* xI, const double* xJ, uint32_t M, uint32_t wI, uint32_t hI, uint32_t wJ, uint32_t hJ,
                      const double* Kpair, const orc_relpose_options* o, orc_relpose_result* r, uint32_t* inliers);
/* every pair of a CSR (omp over pairs); out[P]; inl_ofs[P+1] / inl (capacity = #putatives): inlier matches of OK pairs */
int64_t orc_relative_poses(const float* const* xys, const uint32_t* widths, const uint32_t* heights, const double* Ks,
                           uint32_t n_views, const uint32_t* pairs, uint64_t P, const uint64_t* put_ofs, const orc_indmatch* put,
                           const orc_relpose_options* o, orc_relpose_result* out, uint64_t* inl_ofs, orc_indmatch* inl,
                           int n_threads);

#ifdef __cplusplus
}
#endif
#endif
