/*
 * oracle.h -- C ABI of the CPU ORACLE.
 *
 * TEST INFRASTRUCTURE ONLY.  This library is a dependency-free CPU restatement of the
 * reference's compute-matches + bundle-adjustment hot path.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (regard3d_b200/, libr3dgpu.so) never links, loads or calls anything in oracle/.
 *
 * PARITY UNPINNED: the arithmetic of the reference path lives in un-vendored OpenMVG 1.4 / Ceres
 * (SURVEY.md sec. 0.2, 8c) and the reference ships no tests, golden vectors or fixtures, so this
 * restatement follows the reference's call sites (src/R3DComputeMatches.cpp:423-491, :2035-2233)
 * plus the published upstream algorithms (SURVEY.md Appendix A).  It is cross-checked against
 * independent implementations (numpy / cv2 / scipy) in tests/, not against reference outputs.
 */
#ifndef R3D_ORACLE_H
#define R3D_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { uint32_t i, j; } orc_indmatch;

/* openMVG::matching::L2<float> / L2<unsigned char> (squared, 4-way unrolled float accumulate). */
float orc_l2_f32(const float* a, const float* b, uint64_t n);
float orc_l2_u8(const uint8_t* a, const uint8_t* b, uint64_t n);

/* ArrayMatcherBruteForce::SearchNeighbours, NN=2.  idx/dist have nq*2 entries.
 * dtype 0 = float32, 1 = uint8.  returns 0 on success, 1 if "false" (n_db < 2 or nq < 1). */
int orc_search_neighbours(const void* db, uint32_t n_db, const void* q, uint32_t nq, uint32_t dim,
                          int dtype, int32_t* idx, float* dist, int n_threads);

/* RegionsMatcherT::MatchDistanceRatio(ratio, regionsJ, out): 2-NN, ratio^2 test, (i,j) dedup,
 * coordinate dedup.  out must hold nq entries; returns the number of matches written. */
int64_t orc_match_distance_ratio(const void* descI, const float* xyI, uint32_t nI,
                                 const void* descJ, const float* xyJ, uint32_t nJ,
                                 uint32_t dim, int dtype, float ratio, orc_indmatch* out,
                                 int n_threads);

/* Matcher_Regions::Match over a pair list (serial I, omp-dynamic J).  descs[v]/xys[v]/ns[v] per
 * view.  Output: CSR -- pair_ofs[P+1] offsets into out (capacity cap).  Pairs with no match have
 * an empty range (the reference does not insert them into the map).  returns total matches or -1. */
int64_t orc_match_pairs(const void* const* descs, const float* const* xys, const uint32_t* ns,
                        uint32_t n_views, uint32_t dim, int dtype,
                        const uint32_t* pairs, uint64_t P, float ratio,
                        uint64_t* pair_ofs, orc_indmatch* out, uint64_t cap, int n_threads);

/* Cascade_Hashing_Matcher_Regions::Match (OpenMVG CASCADE_HASHING_L2, SURVEY.md A.8; BASELINE config 4): same
 * arguments and output as orc_match_pairs.  orc_cascade_projections: the (dim + 60) x dim projection table. */
int64_t orc_cascade_match_pairs(const void* const* descs, const float* const* xys, const uint32_t* ns,
                                uint32_t n_views, uint32_t dim, int dtype,
                                const uint32_t* pairs, uint64_t P, float ratio,
                                uint64_t* pair_ofs, orc_indmatch* out, uint64_t cap, int n_threads);
void orc_cascade_projections(uint32_t dim, float* out);

/* IndMatchDecorator<float>::getDeduplicated on an (i,j)-sorted list, in place; returns new count. */
int64_t orc_coord_dedup(orc_indmatch* m, int64_t n, const float* xyI, const float* xyJ);

/* ---- file formats (SURVEY.md Appendix B) ---- */
int orc_save_feat(const char* path, const float* xyso /* n x 4 */, uint32_t n);
int orc_load_feat(const char* path, float* xyso, uint32_t cap, uint32_t* n);
int orc_save_desc_f32(const char* path, const float* d, uint64_t n, uint32_t dim);
int orc_load_desc_f32(const char* path, float* d, uint64_t cap_rows, uint32_t dim, uint64_t* n);
int orc_save_matches_txt(const char* path, const uint32_t* pairs, uint64_t P,
                         const uint64_t* pair_ofs, const orc_indmatch* m);

/* ---- AC-RANSAC fundamental filter (SURVEY.md A.4-A.6) ---- */
/* xI,xJ: M x 2 doubles (pixel coords of the putative matches).  inliers: capacity M.
 * returns number of inliers (0 if the pair is rejected: nfa>=0 or #inliers <= 17.5). */
int64_t orc_acransac_F(const double* xI, const double* xJ, uint32_t M,
                       uint32_t wI, uint32_t hI, uint32_t wJ, uint32_t hJ,
                       double precision_px, uint32_t max_iter,
                       uint32_t* inliers, double* F_out /*9, may be null*/,
                       double* info /* [0]=minNFA [1]=errorMax(px) [2]=iterations run; may be null */);

/* geometric filter over a pair CSR (omp over pairs).  out CSR like orc_match_pairs. */
int64_t orc_filter_pairs_F(const float* const* xys, const uint32_t* widths, const uint32_t* heights,
                           uint32_t n_views, const uint32_t* pairs, uint64_t P,
                           const uint64_t* put_ofs, const orc_indmatch* put,
                           double precision_px, uint32_t max_iter,
                           uint64_t* out_ofs, orc_indmatch* out, int n_threads);

/* homography variants (GeometricFilter_HMatrix_AC: 4-point DLT, asymmetric transfer error) */
int64_t orc_acransac_H(const double* xI, const double* xJ, uint32_t M, uint32_t wI, uint32_t hI, uint32_t wJ, uint32_t hJ,
                       double precision_px, uint32_t max_iter, uint32_t* inliers, double* H_out, double* info);
int64_t orc_filter_pairs_H(const float* const* xys, const uint32_t* widths, const uint32_t* heights,
                           uint32_t n_views, const uint32_t* pairs, uint64_t P,
                           const uint64_t* put_ofs, const orc_indmatch* put,
                           double precision_px, uint32_t max_iter,
                           uint64_t* out_ofs, orc_indmatch* out, int n_threads);
int orc_four_point(const double* x1 /*4x2*/, const double* x2 /*4x2*/, double* H /*9*/);

/* essential variants (GeometricFilter_EMatrix_AC: 5-point on bearing vectors, one-sided epipolar distance in pixels).
 * Kpair = f1, ppx1, ppy1, f2, ppx2, ppy2 ; Ks = n_views x (f, ppx, ppy), f <= 0: no pinhole intrinsic.
 * F_out = K2^-T E K1^-1 of the best model. */
int64_t orc_acransac_E(const double* xI, const double* xJ, uint32_t M, uint32_t wI, uint32_t hI, uint32_t wJ, uint32_t hJ,
                       const double* Kpair, double precision_px, uint32_t max_iter, uint32_t* inliers, double* F_out,
                       double* info);
int64_t orc_filter_pairs_E(const float* const* xys, const uint32_t* widths, const uint32_t* heights, const double* Ks,
                           uint32_t n_views, const uint32_t* pairs, uint64_t P,
                           const uint64_t* put_ofs, const orc_indmatch* put,
                           double precision_px, uint32_t max_iter,
                           uint64_t* out_ofs, orc_indmatch* out, int n_threads);
/* 5-point essential solver on bearing vectors (Nister / Stewenius): returns #models (<= 10), E[k*9..] row-major,
 * b2^T E b1 = 0 */
int orc_five_point(const double* b1 /*5x3*/, const double* b2 /*5x3*/, double* E /*90*/);

/* 7-point solver on (already normalised) points: returns #models, F[k*9..] row-major. */
int orc_seven_point(const double* x1 /*7x2*/, const double* x2 /*7x2*/, double* F /*27*/);

/* ---- bundle adjustment (SURVEY.md A.7) ---- */
typedef struct {
  uint32_t n_cams, n_pts, n_intr;
  uint64_t n_obs;
  double* poses;        /* n_cams x 6: angle-axis(3), t(3); X_cam = R X + t */
  double* intrinsics;   /* n_intr x 6: f, ppx, ppy, k1, k2, k3 */
  double* points;       /* n_pts x 3 */
  const uint32_t* obs_cam; const uint32_t* obs_pt; /* n_obs */
  const uint32_t* cam_intr;                         /* n_cams: intrinsic group of each camera */
  const double* obs_xy;                             /* n_obs x 2 */
  /* optional (NULL / 0 = radial K3, no priors) */
  const uint8_t* intr_model;     /* n_intr: openMVG EINTRINSIC 1..5 */
  const double* intrinsics_ext;  /* n_intr x 2: Brown t1 t2 / fisheye k4 (held fixed) */
  uint32_t n_priors;             /* pose-centre priors (ViewPriors) */
  const uint32_t* prior_cam; const double* prior_center; const double* prior_weight; /* n_priors [x 3] */
} orc_ba_problem;

typedef struct {
  uint32_t max_iterations;     /* Ceres max_num_iterations (500 in the reference config) */
  double huber_a;              /* HuberLoss(a): a = Square(4.0) = 16 ; <=0 -> trivial loss */
  int refine_intrinsics;       /* ADJUST_ALL (1) or NONE (0) */
  double function_tolerance, gradient_tolerance, parameter_tolerance;
  double initial_radius;       /* 1e4 */
  int n_threads;
  double prior_huber_a;        /* HuberLoss(a) of the pose-centre prior blocks; <= 0 trivial */
} orc_ba_options;

typedef struct {
  uint32_t iterations, successful_steps;
  double initial_cost, final_cost;
  int termination;             /* 0 max iters, 1 function tol, 2 gradient tol, 3 parameter tol, 4 failure */
  double seconds_total, seconds_linear;
} orc_ba_summary;

int orc_bundle_adjust(orc_ba_problem* p, const orc_ba_options* o, orc_ba_summary* s,
                      double* cost_trace /* max_iterations+1 or null */);
/* residual (2) and Jacobian (2 x 15: intrinsics 0..5, pose 6..11, point 12..14) of one observation
 * by forward-mode autodiff -- test hook that pins the GPU's analytic derivatives. */
void orc_ba_jacobian(const double* intr, const double* pose, const double* X, const double* obs, double* r, double* J);
void orc_ba_jacobian_model(int model, const double* intr, const double* ext, const double* pose, const double* X,
                           const double* obs, double* r, double* J);
/* pose-centre prior block by autodiff: r[3], J[3 x 6] */
void orc_ba_prior(const double* pose, const double* center, const double* weight, double* r, double* J);
/* OpenMVGHelper::calculateResiduals twin: |residual| per coordinate, 2 per obs. */
void orc_ba_residuals(const orc_ba_problem* p, double* res /* n_obs x 2 */);

/* ---- steps either side of BA (SURVEY.md 8f-3): tracks, triangulation from known poses, outlier checks ---- */
int64_t orc_tracks_build(const uint32_t* pairs, uint64_t P, const uint64_t* pair_ofs, const orc_indmatch* m, uint32_t min_length,
                         uint32_t* track_ids, uint64_t* track_ofs, uint32_t* views, uint32_t* feats, uint64_t cap_tracks,
                         uint64_t cap_nodes);
void orc_triangulate_landmarks(uint32_t n_lm, const uint64_t* obs_ofs, const uint32_t* obs_cam, const double* obs_xy,
                               const double* poses, const uint32_t* cam_intr, const double* intrinsics, const uint8_t* intr_model,
                               const double* intrinsics_ext, double* X, uint8_t* ok);
void orc_landmark_checks(uint32_t n_lm, const uint64_t* obs_ofs, const uint32_t* obs_cam, const double* obs_xy, const double* poses,
                         const uint32_t* cam_intr, const double* intrinsics, const uint8_t* intr_model, const double* intrinsics_ext,
                         const double* X, double thr_px, uint8_t* keep_obs, double* max_angle);

int orc_num_threads(void);
#ifdef __cplusplus
}
#endif
#endif
