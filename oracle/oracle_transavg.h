/*
 * oracle_transavg.h -- C ABI of the CPU ORACLE of the translation-averaging step (liboracle_transavg.so,
 * oracle/transavg.mk).  TEST INFRASTRUCTURE ONLY, like oracle.h: it links liboracle_rotavg.so for the bi-edge-connected
 * component and the dense Cholesky, and liboracle_relpose.so for Ceres' rotation conversions.
 */
#ifndef R3D_ORACLE_TRANSAVG_H
#define R3D_ORACLE_TRANSAVG_H
#include "oracle_relpose.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- global translations (GlobalSfM_Translation_AveragingSolver, L2 chordal / soft-L1) ---- */
typedef struct {
  int method;                  /* 2 L2 chordal ; 3 soft-L1 ; 1 L1 -> -5 */
  double softl1_loss;          /* 0.01 */
  orc_ba_options lm;           /* max_iterations / function_tolerance 0: the method's; n_threads unused (the call's) */
} orc_transavg_options;
/* same layout as r3d_transavg_summary (include/r3dgpu.h) */
typedef struct {
  int success;
  uint64_t n_edges, n_kept_edges;
  uint32_t n_kept_views;
  uint32_t lm_iterations, lm_successful_steps;
  int lm_termination;
  double lm_initial_cost, lm_final_cost;
  double ms_solve, ms_device_total, ms_host;
} orc_transavg_summary;
/* the whole step; inputs and outputs as r3d_translation_averaging.  0, -1 invalid, -5 unsupported */
int orc_translation_averaging(const orc_relpose_result* rel, uint64_t n_rel, const uint8_t* edge_use, const double* rotations,
                              const uint8_t* rot_kept, uint32_t n_views, const orc_transavg_options* o, double* centers,
                              double* translations, uint8_t* view_kept, uint8_t* edge_kept, orc_transavg_summary* s,
                              int n_threads);
/* one edge's residual (3) and Jacobian (3 x 7: x_I, x_J, s; row-major) before the loss, by the jets of the solver.
 * edata: chordal u = -R_J^T t_IJ / |t_IJ| (3); soft-L1 the angle-axis of R_IJ (3) then t_IJ / |t_IJ| (3) */
void orc_transavg_edge(int method, const double* xi, const double* xj, double s, const double* edata, double* res, double* jac);
/* ceres::SoftLOneLoss(a) at s = |r|^2: returns rho, *rho1 = rho' */
double orc_softl1_rho(double sq, double a, double* rho1);

#ifdef __cplusplus
}
#endif
#endif
