/*
 * oracle_rotavg.h -- C ABI of the CPU ORACLE of the rotation-averaging step (liboracle_rotavg.so, oracle/rotavg.mk).
 * TEST INFRASTRUCTURE ONLY, like oracle.h: it links liboracle_relpose.so for the Jacobi SVD and Ceres' rotation
 * conversions that the relative-pose oracle already restates.
 */
#ifndef R3D_ORACLE_ROTAVG_H
#define R3D_ORACLE_ROTAVG_H
#include "oracle_relpose.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- global rotations (GlobalSfM_Rotation_AveragingSolver::Run, ROTATION_AVERAGING_L2) ---- */
typedef struct {
  int method;                  /* 0 L2 ; 1 L1 -> -5 */
  double max_angular_error_deg;/* 5.0 */
  int refine;                  /* L2RotationAveraging_Refine */
  orc_ba_options lm;           /* huber_a <= 0: trivial loss; n_threads unused (the call's n_threads) */
} orc_rotavg_options;
/* same layout as r3d_rotavg_summary (include/r3dgpu.h) */
typedef struct {
  int success;
  uint64_t n_edges, n_triplets, n_valid_triplets, n_kept_edges;
  uint32_t n_kept_views, init_iterations;
  uint32_t lm_iterations, lm_successful_steps;
  int lm_termination;
  double lm_initial_cost, lm_final_cost;
  double ms_triplets, ms_init, ms_refine, ms_device_total, ms_host;
} orc_rotavg_summary;
/* the whole step on an array of relative poses; outputs as r3d_rotation_averaging.  0, -1 invalid, -5 unsupported */
int orc_rotation_averaging(const orc_relpose_result* rel, uint64_t n_rel, uint32_t n_views, const orc_rotavg_options* o,
                           double* rotations, uint8_t* view_kept, uint8_t* edge_kept, uint32_t* edge_support,
                           orc_rotavg_summary* s, int n_threads);
/* the triplet error in degrees (float) of R_ij, R_jk, R_ik (canonical orientations) */
float orc_rotavg_cycle_error(const double* Rij, const double* Rjk, const double* Rik);
/* every triangle {i < j < k} of the edges ij (E x 2, any orientation; R: E x 9, R_ij of the pair (min, max)): tri
 * (cap x 3 view ids), err, valid (err < thr); returns the count */
int64_t orc_rotavg_triplets(const uint32_t* ij, const double* R, uint64_t E, uint32_t n_views, float thr, uint32_t* tri,
                            float* err, uint8_t* valid, uint64_t cap);
/* kept[v] = 1 for the views of the largest 2-edge-connected component; returns their count */
int orc_largest_biedge_component(const uint32_t* ij, uint64_t E, uint32_t n_views, uint8_t* kept);
/* the linear step on local ids (ab: E x 2, a < b; R: R_ab): M (3m x 3m, may be NULL) and the orthonormal basis Q (3m x 3)
 * of its 3 smallest eigenvectors; returns the inverse iterations (0: M + sigma I not positive definite) */
uint32_t orc_rotavg_l2_subspace(const uint32_t* ab, const double* R, uint64_t E, uint32_t m, double* M, double* Q, int n_threads);

#ifdef __cplusplus
}
#endif
#endif
