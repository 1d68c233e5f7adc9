/*
 * r3dgpu.h -- C ABI of libr3dgpu.so: the H100 (sm_90a) replacement of Regard3D's compute-matches
 * hot path and the downstream bundle-adjustment solve.
 *
 * Every entry point names the reference interface it replaces (paths relative to the Regard3D
 * tree, rhiestan/Regard3D @ 2822275).  The reference has no FFI of its own: the binding a
 * maintainer adds is the C++ shim in regard3d_b200/csrc/R3DComputeMatches_b200.{h,cpp} (same
 * class name / method set as src/R3DComputeMatches.h:30-74); see INTEGRATION.md.
 *
 * Conventions: plain pointers + sizes, host memory in and out, no C++/CUDA/torch types.
 * Return value: 0 = R3D_OK, negative = error (r3d_last_error() gives the text).  There is NO CPU
 * fallback: without a usable sm_90 device r3d_create() fails with R3D_ERR_NO_DEVICE.
 * Threading: a context may be used from any one thread at a time (the reference calls
 * computeMatches() on one dedicated wxThread: src/threads/R3DComputeMatchesThread.cpp:91-103).
 */
#ifndef R3DGPU_H
#define R3DGPU_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define R3D_ABI_VERSION 3

typedef enum {
  R3D_OK = 0,
  R3D_ERR_INVALID = -1,      /* bad argument */
  R3D_ERR_CUDA = -2,         /* a CUDA runtime / driver call failed */
  R3D_ERR_NOMEM = -3,
  R3D_ERR_IO = -4,           /* file could not be read / written */
  R3D_ERR_UNSUPPORTED = -5,  /* e.g. descriptor range outside what the fp16 operand can hold */
  R3D_ERR_NO_DEVICE = -6     /* no sm_90 GPU: the library never falls back to the CPU */
} r3d_status;

typedef enum { R3D_F32 = 0, R3D_U8 = 1 } r3d_dtype;

/* openMVG::matching::IndMatch{i_,j_}: i_ indexes the FIRST image of the pair, j_ the second
 * (consumer: src/threads/PreviewGeneratorThread.cpp:373-390). */
typedef struct { uint32_t i, j; } r3d_indmatch;

typedef struct r3d_ctx r3d_ctx;
/* openMVG::matching::PairWiseMatches = std::map<Pair, IndMatches> (opaque, host memory). */
typedef struct r3d_matches r3d_matches;

/* ---- context ------------------------------------------------------------------------------- */
/* One context drives the listed CUDA devices (one worker + stream set per device; pairs shard
 * across them without any collective).  bench.py uses one process per GPU, i.e. n_devices = 1.
 * Replaces: construction of R3DComputeMatches (src/threads/R3DComputeMatchesThread.cpp:91). */
int r3d_create(const int* device_ids, int n_devices, r3d_ctx** out);
void r3d_destroy(r3d_ctx* ctx);
const char* r3d_last_error(const r3d_ctx* ctx); /* ctx may be NULL: last global error */
int r3d_abi_version(void);

/* ---- regions ------------------------------------------------------------------------------- */
/* Replaces Regions_Provider::load (src/R3DComputeMatches.cpp:2040) for one view:
 * desc = Regions::DescriptorRawData() (n x dim row-major, float32 or uint8; Regard3D's native
 * type is Scalar_Regions<SIOPointFeature,float,144>, src/Regard3DFeatures.h:42-48),
 * xy = feature positions (n x 2 float32, from the .feat file; may be NULL if no coordinate
 * de-duplication / geometric filtering will be requested).  Data is copied. */
int r3d_upload_regions(r3d_ctx* ctx, uint32_t view_id, const void* desc, uint32_t n, uint32_t dim,
                       int dtype, const float* xy);
int r3d_clear_regions(r3d_ctx* ctx);

/* ---- descriptors (SURVEY.md 8f-1: the stage that feeds the .desc files) ------------------------------ */
/* cv::KeyPoint as Regard3D uses it: position, size = diameter, angle in degrees. */
typedef struct { float x, y, size, angle; } r3d_keypoint;
/* Replaces Regard3DFeatures::extractLIOPFeatures (src/Regard3DFeatures.cpp:719-861) for one image: per keypoint a
 * 41x41 patch (cv::warpAffine with the inverse map of :766-800, cv::GaussianBlur sigma 1.2) and its LIOP descriptor
 * r3d_vl_liopdesc_process [src/thirdparty/liop/vl_liop.c:434-575] (4 neighbours, 6 spatial bins, radius 6 -> 144
 * floats, unit L2 norm).  image: height x width float32 row-major (openMVG::image::Image<float>, cv::eigen2cv);
 * kp_size_factor: Regard3DFeatures::getKpSizeFactor (:691-716; 8 for AKAZE / Fast-AKAZE); desc_out: n x 144, in
 * keypoint order (the reference appends in thread-completion order, :838-851). */
int r3d_liop_describe(r3d_ctx* ctx, const float* image, uint32_t width, uint32_t height,
                      const r3d_keypoint* keypoints, uint32_t n, float kp_size_factor, float* desc_out);
/* Diagnostics: the descriptor function alone (vl_liop.c:434-575) on n ready 41x41 float32 patches. */
int r3d_debug_liop_process(r3d_ctx* ctx, const float* patches, uint32_t n, float* desc_out);

/* ---- putative matching --------------------------------------------------------------------- */
#define R3D_MATCH_DEFAULT 0u
#define R3D_MATCH_EXACT_SCAN 1u   /* skip the tensor-core candidate pass: CUDA-core exact scan only */
#define R3D_MATCH_NO_COORD_DEDUP 2u /* skip IndMatchDecorator (for callers without positions) */
#define R3D_MATCH_CASCADE_HASHING 8u /* OpenMVG CASCADE_HASHING_L2 (BASELINE config 4) instead of the exhaustive 2-NN:
                                   * approximate by construction, bit-identical to the CPU restatement of the algorithm */
#define R3D_MATCH_MUTUAL_NN 4u    /* OFF by default and NOT reference behaviour (MatchDistanceRatio has no cross-check):
                                   * keep (i, j) only if j is also i's nearest neighbour among J's descriptors */

/* Replaces Matcher_Regions(fDistRatio, BRUTE_FORCE_L2)::Match(regions_provider, pairs, out)
 * (src/R3DComputeMatches.cpp:2039, :2048; loop shape :437-488): for every pair (I,J): 2-NN of each
 * J descriptor in I under squared L2, keep iff d1 < ratio^2 * d2, IndMatch(i in I, j in J),
 * (i,j) de-duplication, coordinate de-duplication.  pairs = P x 2 view ids.  Pairs without
 * matches are absent from the result, like in the reference's map. */
int r3d_match_pairs(r3d_ctx* ctx, const uint32_t* pairs, uint64_t n_pairs, float dist_ratio,
                    uint32_t flags, r3d_matches** out);

/* R3D_MATCH_CASCADE_HASHING replaces Cascade_Hashing_Matcher_Regions::Match (OpenMVG matching_image_collection, the
 * matcher BASELINE config 4 names; Regard3D's own GUI never selects it, src/R3DComputeMatches.cpp:2035-2062).  Its hash
 * codes depend on the zero-mean descriptor of ALL views of the matching job, so a job that is split over several
 * r3d_match_pairs calls (ranks, shards) declares its views once: r3d_cascade_prepare hashes the given views (already
 * uploaded) under their common zero-mean descriptor; later R3D_MATCH_CASCADE_HASHING calls whose pairs stay inside
 * that set reuse the tables.  Without it every call hashes the views of its own pair list (= one call is one job, the
 * reference's behaviour).  Views of more than 65536 features or dimension > 256: R3D_ERR_UNSUPPORTED. */
int r3d_cascade_prepare(r3d_ctx* ctx, const uint32_t* view_ids, uint32_t n_views);

/* Replaces openMVG::matching::ArrayMatcher<float,L2>::SearchNeighbours(query, nbQuery, &idx, &dist,
 * NN=2) -- the plug-in API Regard3D implements in src/utils/matcher_hnsw.h:133-191 -- with the
 * database = regions of view_db (ArrayMatcher::Build, :53-68) and queries = regions of view_query.
 * idx / dist: n_query x 2, ascending exact squared distance (float accumulate, upstream order). */
int r3d_search_neighbours(r3d_ctx* ctx, uint32_t view_db, uint32_t view_query, int32_t* idx,
                          float* dist);

/* ---- PairWiseMatches accessors ------------------------------------------------------------- */
uint64_t r3d_matches_num_pairs(const r3d_matches* m);
uint64_t r3d_matches_total(const r3d_matches* m);
/* k-th pair in std::map order (sorted by I, then J). */
int r3d_matches_get_pair(const r3d_matches* m, uint64_t k, uint32_t* I, uint32_t* J,
                         const r3d_indmatch** matches, uint64_t* count);
/* Build a PairWiseMatches from CSR arrays (pair_ofs has n_pairs+1 entries). */
int r3d_matches_from_csr(const uint32_t* pairs, uint64_t n_pairs, const uint64_t* pair_ofs,
                         const r3d_indmatch* matches, r3d_matches** out);
/* Flat copy of the map in std::map order: pairs_out 2 x num_pairs view ids, ofs_out num_pairs + 1 prefix offsets,
 * matches_out r3d_matches_total() entries; any output may be NULL.  This is what a per-GPU process ships when the
 * pair list is sharded over ranks and the PairWiseMatches map is re-assembled on one of them (SURVEY.md 8e:
 * "results concatenated on host in pair order"; the reference's map insert is src/R3DComputeMatches.cpp:483-486). */
int r3d_matches_export_csr(const r3d_matches* m, uint32_t* pairs_out, uint64_t* ofs_out,
                           r3d_indmatch* matches_out);
void r3d_free_matches(r3d_matches* m);
/* matching::Save / matching::Load, text format (src/R3DComputeMatches.cpp:2064, :2120;
 * SURVEY.md Appendix B.3). */
int r3d_save_matches_txt(const r3d_matches* m, const char* path);
int r3d_load_matches_txt(const char* path, r3d_matches** out);

/* matching::Save / matching::Load as the reference calls them: the extension picks the format -- ".txt" (above) or
 * ".bin" = cereal PortableBinary of std::map<Pair, std::vector<IndMatch>> (SURVEY.md App. B.3; layout restated in
 * regard3d_b200/csrc/sfm_data_io.cpp). */
int r3d_save_matches_bin(const r3d_matches* m, const char* path);
int r3d_load_matches_bin(const char* path, r3d_matches** out);
int r3d_save_matches(const r3d_matches* m, const char* path);
int r3d_load_matches(const char* path, r3d_matches** out);

/* ---- sfm_data.bin (SURVEY.md App. B.4) ------------------------------------------------------------------------
 * openMVG::sfm::SfM_Data as the reference stores it: cereal PortableBinary "sfm_data.bin", written by
 * R3DProject::writeSfmData (src/R3DProject.cpp:1118-1306: views / view priors + intrinsics), read by
 * R3DComputeMatches::computeMatches (src/R3DComputeMatches.cpp:1755) and R3DTriangulationThread
 * (src/threads/R3DTriangulationThread.cpp:403), written back with poses + structure (:453-455).  Opaque handle +
 * plain-struct accessors; maps are walked in key order (k-th element). */
typedef struct r3d_sfm_data r3d_sfm_data;
/* openMVG::sfm::ESfM_Data */
#define R3D_SFM_VIEWS 1u
#define R3D_SFM_EXTRINSICS 2u
#define R3D_SFM_INTRINSICS 4u
#define R3D_SFM_STRUCTURE 8u
#define R3D_SFM_CONTROL_POINTS 16u
#define R3D_SFM_ALL 31u
/* openMVG::cameras::EINTRINSIC (the `cameraModel` argument of computeMatches, src/R3DProject.cpp:1167-1191) */
#define R3D_CAM_PINHOLE 1
#define R3D_CAM_PINHOLE_RADIAL1 2
#define R3D_CAM_PINHOLE_RADIAL3 3
#define R3D_CAM_PINHOLE_BROWN 4
#define R3D_CAM_PINHOLE_FISHEYE 5
typedef struct {
  uint32_t id_view, id_intrinsic, id_pose, width, height;
  const char* local_path;  /* folder part of View::s_Img_path */
  const char* filename;    /* file part */
  int has_prior;           /* openMVG::sfm::ViewPriors with b_use_pose_center_ (GPS; src/R3DProject.cpp:1194-1220) */
  double center_weight[3], pose_center[3];
} r3d_sfm_view;
typedef struct {
  uint32_t id;
  int model;               /* R3D_CAM_* */
  uint32_t width, height;
  double focal, ppx, ppy;
  double disto[5];         /* K1: k1 | K3: k1 k2 k3 | Brown T2: k1 k2 k3 t1 t2 | fisheye: k1 k2 k3 k4 */
} r3d_sfm_intrinsic;
typedef struct { uint32_t id; double rotation[9]; double center[3]; } r3d_sfm_pose;  /* geometry::Pose3: R row-major, C */
typedef struct { uint32_t id_view, id_feat; double x[2]; } r3d_sfm_observation;
int r3d_sfm_data_create(r3d_sfm_data** out);
void r3d_sfm_data_free(r3d_sfm_data* sd);
int r3d_sfm_data_load(const char* path, r3d_sfm_data** out);                       /* Load(sfm_data, path, ALL) */
int r3d_sfm_data_save(const r3d_sfm_data* sd, const char* path, uint32_t parts);   /* Save(sfm_data, path, parts) */
const char* r3d_sfm_root_path(const r3d_sfm_data* sd);
int r3d_sfm_set_root_path(r3d_sfm_data* sd, const char* root_path);
uint32_t r3d_sfm_num_views(const r3d_sfm_data* sd);
uint32_t r3d_sfm_num_intrinsics(const r3d_sfm_data* sd);
uint32_t r3d_sfm_num_poses(const r3d_sfm_data* sd);
uint32_t r3d_sfm_num_landmarks(const r3d_sfm_data* sd, int control_points);
int r3d_sfm_add_view(r3d_sfm_data* sd, const r3d_sfm_view* v);                     /* strings are copied */
int r3d_sfm_get_view(const r3d_sfm_data* sd, uint32_t k, r3d_sfm_view* out);       /* strings owned by sd */
int r3d_sfm_add_intrinsic(r3d_sfm_data* sd, const r3d_sfm_intrinsic* in);
int r3d_sfm_get_intrinsic(const r3d_sfm_data* sd, uint32_t k, r3d_sfm_intrinsic* out);
int r3d_sfm_add_pose(r3d_sfm_data* sd, const r3d_sfm_pose* p);
int r3d_sfm_get_pose(const r3d_sfm_data* sd, uint32_t k, r3d_sfm_pose* out);
int r3d_sfm_add_landmark(r3d_sfm_data* sd, int control_point, uint32_t id, const double X[3],
                         const r3d_sfm_observation* obs, uint32_t n_obs);
int r3d_sfm_get_landmark(const r3d_sfm_data* sd, int control_point, uint32_t k, uint32_t* id, double X[3],
                         r3d_sfm_observation* obs, uint32_t obs_cap, uint32_t* n_obs);

/* ---- geometric filtering ------------------------------------------------------------------- */
typedef enum { R3D_MODEL_F = 0, R3D_MODEL_E = 1, R3D_MODEL_H = 2 } r3d_model;
/* One entry per view id (sfm_data views + their intrinsics).  focal / ppx / ppy: pinhole K of the view as
 * R3DProject builds it (src/R3DProject.cpp:1149-1159: focal = max(w,h) * focal_mm / sensor_width, else
 * 1.1 * max(w,h); pp = (w/2, h/2)); only the essential filter reads them, focal <= 0 = "no valid pinhole
 * intrinsic" (the pair is dropped, as GeometricFilter_EMatrix_AC does). */
typedef struct { uint32_t width, height; double focal, ppx, ppy; } r3d_view_info;

/* Replaces ImageCollectionGeometricFilter::Robust_model_estimation(
 *   GeometricFilter_FMatrix_AC(precision_px = 4.0, max_iter = 2048), putative, false)
 * + Get_geometric_matches() (src/R3DComputeMatches.cpp:2099-2115).  Uses the positions uploaded
 * with r3d_upload_regions.  views[v] = image size of view v (sfm_data views).
 * R3D_MODEL_H: GeometricFilter_HMatrix_AC(4.0, 2048) (src/R3DComputeMatches.cpp:2215-2219; 4-point DLT,
 * asymmetric transfer error, point-to-point a-contrario model).
 * R3D_MODEL_E: GeometricFilter_EMatrix_AC(4.0, 2048) (:2169-2171; Nister/Stewenius 5-point solver on bearing
 * vectors, <= 10 models per sample, one-sided epipolar distance of F = K2^-T E K1^-1 in pixels). The
 * poor-overlap post-filter of :2173-2191 belongs to computeMatches() and is applied by r3d_compute_matches. */
int r3d_filter_pairs(r3d_ctx* ctx, int model, double precision_px, uint32_t max_iter,
                     const r3d_matches* putative, const r3d_view_info* views, uint32_t n_views,
                     r3d_matches** out);

/* ---- bundle adjustment --------------------------------------------------------------------- */
/* Replaces openMVG::sfm::Bundle_Adjustment_Ceres::Adjust as driven by the SfM engines' Process()
 * (src/threads/R3DTriangulationThread.cpp:441, :512, :250).  Default camera model: pinhole radial-K3 (chosen at :398,
 * built at src/R3DProject.cpp:1177-1180); the four other models the reference can store are selected per intrinsic
 * group with intr_model.  Tracks may have any length. */
typedef struct {
  uint32_t n_cams, n_pts, n_intr;
  uint64_t n_obs;
  double* poses;       /* n_cams x 6: angle-axis, t ; X_cam = R X + t          (in/out) */
  double* intrinsics;  /* n_intr x 6: f, ppx, ppy, k1, k2, k3                  (in/out) */
  double* points;      /* n_pts x 3                                            (in/out) */
  const uint32_t* obs_cam;   /* n_obs */
  const uint32_t* obs_pt;    /* n_obs */
  const uint32_t* cam_intr;  /* n_cams: intrinsic group of each camera */
  const double* obs_xy;      /* n_obs x 2 */
  /* --- ABI 3 (all optional: NULL / 0 = round-1 behaviour) --- */
  const uint8_t* intr_model; /* n_intr: camera model of each group, R3D_CAM_* (src/R3DProject.cpp:1167-1191); NULL = radial K3.
                              * intrinsics[g] = f, ppx, ppy, then the model's first three distortion coefficients
                              * (pinhole: none, K1: k1, K3 / Brown: k1 k2 k3, fisheye: k1 k2 k3); slots a model does not
                              * own are ignored and never change */
  const double* intrinsics_ext; /* n_intr x 2 or NULL: Brown T2: t1 t2, fisheye: k4 -- read, HELD FIXED by the solve
                              * (intrinsic blocks of the reduced camera system are 6 wide) */
  uint32_t n_priors;         /* pose-centre priors = openMVG ViewPriors with b_use_pose_center_ (GPS) */
  const uint32_t* prior_cam; /* n_priors: camera (pose) index */
  const double* prior_center;/* n_priors x 3 */
  const double* prior_weight;/* n_priors x 3 (ViewPriors::center_weight_) */
} r3d_ba_problem;

typedef struct {
  uint32_t max_iterations;   /* 500 */
  double huber_a;            /* HuberLoss(Square(4.0)) -> 16 ; <= 0: trivial loss */
  int refine_intrinsics;     /* Intrinsic_Parameter_Type ADJUST_ALL (1) / NONE (0), R3DTriangulationThread.cpp:429-432 */
  double function_tolerance; /* 1e-6 */
  double gradient_tolerance; /* 1e-10 */
  double parameter_tolerance;/* 1e-8 */
  double initial_radius;     /* 1e4 */
  double prior_huber_a;      /* ABI 3: HuberLoss(a) of the pose-centre prior blocks (OpenMVG: Square(pose_center_robust_
                              * fitting_error)); <= 0: trivial loss */
} r3d_ba_options;

typedef struct {
  uint32_t iterations, successful_steps;
  double initial_cost, final_cost;
  int termination;           /* 0 max iters, 1 function tol, 2 gradient tol, 3 parameter tol, 4 failure */
  double seconds_total, seconds_linear;
  double seconds_setup;      /* validation, CSR build, uploads (inside seconds_total) */
} r3d_ba_summary;

void r3d_ba_default_options(r3d_ba_options* o);
int r3d_bundle_adjust(r3d_ctx* ctx, r3d_ba_problem* io, const r3d_ba_options* opt,
                      r3d_ba_summary* summary, double* cost_trace /* max_iterations+1 or NULL */);

/* openMVG::sfm::Bundle_Adjustment_Ceres::Adjust(SfM_Data&, Optimize_Options) on the SfM_Data container itself: poses
 * (R, C) <-> angle-axis | t, one parameter block per intrinsic id in its own camera model, landmarks; refined values are
 * written back into sd.  solver.refine_intrinsics = Intrinsic_Parameter_Type ADJUST_ALL / NONE; use_motion_priors adds
 * one pose-centre block per ViewPriors view (sfmEngine.Set_Use_Motion_Prior, R3DTriangulationThread.cpp:433).  The C++
 * adaptor with the reference's class shape is regard3d_b200/csrc/Bundle_Adjustment_b200.h. */
typedef struct {
  r3d_ba_options solver;
  int use_motion_priors;
} r3d_sfm_ba_options;
void r3d_sfm_ba_default_options(r3d_sfm_ba_options* o);
int r3d_sfm_bundle_adjust(r3d_ctx* ctx, r3d_sfm_data* sd, const r3d_sfm_ba_options* opt, r3d_ba_summary* summary);

/* ---- relative pose of every image pair (global SfM) ------------------------------------------ */
#define R3D_RELPOSE_OK 0
#define R3D_RELPOSE_TOO_FEW 1        /* <= 5 matches */
#define R3D_RELPOSE_NO_INTRINSIC 2   /* focal <= 0 in either view */
#define R3D_RELPOSE_NO_MODEL 3       /* AC-RANSAC: minNFA >= 0 or fewer than 2.5 * 5 inliers */
#define R3D_RELPOSE_CHEIRALITY 4     /* no motion of E puts an inlier in front of both cameras */
typedef struct {
  double precision_px;       /* 2.5: RelativePose_Info::initial_residual_tolerance = Square(2.5) */
  uint32_t max_iter;         /* 256 */
  int refine;                /* 1: bRefine_using_BA, the two-view bundle adjustment of each pair */
  r3d_ba_options ba;         /* refine_intrinsics must be 0 (the pair's intrinsics stay fixed); prior_huber_a unused */
} r3d_relpose_options;
void r3d_relpose_default_options(r3d_relpose_options* o);  /* 2.5, 256, 1, r3d_ba_default_options with intrinsics fixed */
typedef struct {
  uint32_t I, J;
  int status;                        /* R3D_RELPOSE_* */
  uint32_t n_inliers;
  double found_residual_precision;   /* AC-RANSAC errorMax, px */
  double E[9];                       /* K2^T F K1 of AC-RANSAC's best model F: the 5-point solver's E up to rounding */
  double rotation[9], translation[3];/* X_J = R X_I + t, R row-major; |t| = 1 before refinement */
  uint32_t ba_iterations, ba_successful_steps;
  int ba_termination;                /* as r3d_ba_summary.termination; -1: not refined.  4 (failure): R, t unrefined */
  double ba_initial_cost, ba_final_cost;
} r3d_relative_pose;
/* Replaces the loop body of GlobalSfMReconstructionEngine_RelativeMotions::Compute_Relative_Rotations (OpenMVG 1.4
 * sfm_global_engine_relative_motions.cpp, reached from src/threads/R3DTriangulationThread.cpp:201-250 on
 * matches.e.txt) for every pair of `matches`: robustRelativePose (AC-RANSAC with the essential adaptor, 5-point solver,
 * precision_px / max_iter), MotionFromEssential + the cheirality test, then the two-view Bundle_Adjustment_Ceres of the
 * pair (both poses and every match's DLT point, intrinsics fixed) and RelativeCameraMotion.  Positions come from
 * r3d_upload_regions; views[v] gives the size and pinhole K of view v (as for R3D_MODEL_E).  out: one entry per pair
 * of `matches`, in map order.  inliers (may be NULL): the AC-RANSAC inliers (residual order) of the OK pairs. */
int r3d_relative_poses(r3d_ctx* ctx, const r3d_matches* matches, const r3d_view_info* views, uint32_t n_views,
                       const r3d_relpose_options* opt, r3d_relative_pose* out, r3d_matches** inliers);
typedef struct {
  double ms_ransac, ms_cheirality, ms_refine, ms_device_total, ms_host;  /* last r3d_relative_poses call */
  uint64_t kernel_launches, ba_iterations;
} r3d_relpose_timing;
int r3d_get_relpose_timing(const r3d_ctx* ctx, r3d_relpose_timing* out);

/* ---- resection: the absolute pose of views from 2D-3D correspondences (incremental SfM's first step) ----------- */
#define R3D_RESECT_OK 0
#define R3D_RESECT_TOO_FEW 1         /* <= 3 correspondences */
#define R3D_RESECT_NO_INTRINSIC 2    /* focal <= 0 (upstream falls back to a 6-point DLT there; not implemented) */
#define R3D_RESECT_NO_MODEL 3        /* AC-RANSAC: minNFA >= 0 or <= 2.5 * 3 inliers */
typedef struct {
  double precision_px;       /* +inf: SfM_Localizer's error_max = infinity (pure a-contrario); finite: the upper bound */
  uint32_t max_iter;         /* 4096 */
  int refine;                /* 1: SfM_Localizer::RefinePose(b_refine_pose = true, b_refine_intrinsic = false) */
  r3d_ba_options ba;         /* the refinement's trust region and Huber loss; refine_intrinsics must be 0 */
} r3d_resection_options;
void r3d_resection_default_options(r3d_resection_options* o);  /* +inf, 4096, 1, r3d_ba_default_options with intrinsics fixed */
typedef struct {
  uint32_t view_id, width, height;
  r3d_sfm_intrinsic intrinsic;       /* any R3D_CAM_* model; focal <= 0: no pinhole intrinsic */
  uint64_t first, count;             /* the view's correspondences in X / x */
} r3d_resection_view;
typedef struct {
  uint32_t view_id;
  int status;                        /* R3D_RESECT_* */
  uint32_t n_inliers;
  double found_residual_precision;   /* AC-RANSAC errorMax, px */
  double rotation[9], center[3], translation[3];     /* X_cam = R X + t, C = -R^T t; refined when refine is set and
                                                      * the solve did not fail, else the AC-RANSAC pose */
  double rotation_ransac[9], translation_ransac[3];  /* the AC-RANSAC model */
  uint32_t lm_iterations, lm_successful_steps;
  int lm_termination;                /* as r3d_ba_summary.termination; -1: not refined */
  double lm_initial_cost, lm_final_cost;
} r3d_resection;
/* Replaces SfM_Localizer::Localize + SfM_Localizer::RefinePose (OpenMVG 1.4 sfm_localizer.cpp; the resection step of
 * both incremental engines, src/threads/R3DTriangulationThread.cpp:416-512) for a batch of views.  Per view: the pixels
 * undistorted once by the inverse of its camera model, AC-RANSAC with the a-contrario adaptor for resection with known K
 * (P3P on bearing vectors, up to 4 models per sample, squared pixel reprojection error of P = K [R | t], point-to-point
 * model log10(pi / (w h))), then Levenberg-Marquardt on the six pose parameters over the inliers, residuals on the
 * original pixels through the full camera model, HuberLoss(ba.huber_a), structure and intrinsics held.
 * X: 3 doubles per correspondence, x: 2 (pixels).  inliers (may be NULL; capacity: every view's count): per view its
 * AC-RANSAC inliers as indices into its correspondences, in residual order; inlier_ofs (n_views + 1; required with
 * inliers, else may be NULL).  Non-finite X or x, an unknown camera model, a view without a size or
 * ba.refine_intrinsics != 0: R3D_ERR_INVALID before anything runs.  Views are spread over the context's devices. */
int r3d_resect_views(r3d_ctx* ctx, const r3d_resection_view* views, uint32_t n_views, const double* X, const double* x,
                     const r3d_resection_options* opt, r3d_resection* out, uint32_t* inliers, uint64_t* inlier_ofs);
/* The same on an SfM_Data: the correspondences of a view are the landmarks of sd.structure that hold an observation of
 * it (X from the landmark, x from the observation, landmark-id order).  view_ids / n: the views to resect; n = 0: every
 * view without a pose.  out: one entry per resected view (capacity n, or the number of views without a pose), in
 * view_ids order (n = 0: view-id order); *n_out (may be NULL) their number.  Every OK view gets a Pose3 (R, C) under its
 * id_pose; nothing else changes.  A view that already has a pose, an unknown view or intrinsic id: R3D_ERR_INVALID. */
int r3d_sfm_resect_views(r3d_ctx* ctx, r3d_sfm_data* sd, const uint32_t* view_ids, uint32_t n,
                         const r3d_resection_options* opt, r3d_resection* out, uint32_t* n_out);
typedef struct {
  double ms_ransac, ms_refine, ms_device_total, ms_host;  /* last r3d_resect_views call; ms_ransac includes the point kernel */
  uint64_t kernel_launches, lm_iterations;
} r3d_resection_timing;
int r3d_get_resection_timing(const r3d_ctx* ctx, r3d_resection_timing* out);

/* ---- global rotations from the relative motions (global SfM, second step) ------------------------------------- */
#define R3D_ROTAVG_L2 0              /* ROTATION_AVERAGING_L2 (src/threads/R3DTriangulationThread.cpp:201) */
#define R3D_ROTAVG_L1 1              /* ROTATION_AVERAGING_L1: R3D_ERR_UNSUPPORTED here, solved by
                                      * r3d_rotation_averaging_l1 */
#define R3D_ROTAVG_MAX_VIEWS 4096    /* kept views above this (a dense 3n x 3n system): R3D_ERR_UNSUPPORTED */
typedef struct {
  int method;                        /* R3D_ROTAVG_L2 */
  double max_angular_error_deg;      /* 5.0: TripletRotationRejection threshold, a triplet is valid iff float(error) < it */
  int refine;                        /* 1: L2RotationAveraging_Refine after the linear initialisation */
  r3d_ba_options lm;                 /* the refinement's trust region; refine_intrinsics and prior_huber_a unused,
                                      * huber_a <= 0: trivial loss (the default) */
} r3d_rotavg_options;
void r3d_rotavg_default_options(r3d_rotavg_options* o);  /* L2, 5.0, 1, r3d_ba_default_options with a trivial loss */
typedef struct {
  int success;                       /* 0: no bi-edge-connected component survived (upstream returns false) */
  uint64_t n_edges;                  /* R3D_RELPOSE_OK entries of the input */
  uint64_t n_triplets, n_valid_triplets;
  uint64_t n_kept_edges;
  uint32_t n_kept_views;
  uint32_t init_iterations;          /* block inverse iterations of the linear initialisation */
  uint32_t lm_iterations, lm_successful_steps;
  int lm_termination;                /* as r3d_ba_summary.termination; -1: not refined */
  double lm_initial_cost, lm_final_cost;
  double ms_triplets, ms_init, ms_refine, ms_device_total, ms_host;
} r3d_rotavg_summary;
/* Replaces GlobalSfMReconstructionEngine_RelativeMotions::Compute_Global_Rotations = GlobalSfM_Rotation_AveragingSolver::
 * Run (OpenMVG 1.4, ROTATION_AVERAGING_L2, reached from src/threads/R3DTriangulationThread.cpp:201-250) on the OK entries
 * of r3d_relative_poses: every OK entry is one edge (I, J) with R_J ~ rotation R_I (X_J = R X_I + t); triplet rotation
 * rejection (a triangle is valid when its cycle R_ki R_jk R_ij is within max_angular_error_deg of the identity; an edge
 * survives when a valid triangle holds it), the largest bi-edge-connected component of the surviving edges, the L2
 * linear initialisation (Martinec-Pajdla), then the non-linear L2 refinement (angle-axis per view, one residual
 * log(R_ij^T R_j R_i^T) per edge).  Gauge: the lowest kept view id gets R = I exactly.  Outputs: rotations n_views x 9
 * (X_cam = R X, row-major; zero for views outside the component), view_kept n_views, edge_kept / edge_support n_rel
 * (may be NULL; support = valid triangles through the edge, 0 for entries that are not OK).  I == J, a view id >=
 * n_views or an unordered pair given twice among the OK entries: R3D_ERR_INVALID.  One global problem: it runs on the
 * context's first device. */
int r3d_rotation_averaging(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                           const r3d_rotavg_options* opt, double* rotations, uint8_t* view_kept, uint8_t* edge_kept,
                           uint32_t* edge_support, r3d_rotavg_summary* summary);
/* ---- global rotations by Regard3D's "L1 rotation averaging (Chatterjee)", ROTATION_AVERAGING_L1 ------------------- */
typedef struct {
  double max_angular_error_deg;      /* 5.0: the same TripletRotationRejection as the L2 method */
  double irls_sigma_deg;             /* 5.0: Geman-McClure scale of the IRLS step (> 0) */
  int l1_max_iterations;             /* 32: L1RA outer iterations (>= 1) */
  int irls_max_iterations;           /* 32: IRLS iterations (>= 0; 0 skips IRLS) */
  double tolerance;                  /* 1e-5: a loop stops when max_v |x_v| (radians) of its last update <= tolerance (> 0) */
} r3d_rotavg_l1_options;
void r3d_rotavg_l1_default_options(r3d_rotavg_l1_options* o);  /* 5.0, 5.0, 32, 32, 1e-5 */
typedef struct {
  int success;                       /* as r3d_rotavg_summary */
  uint64_t n_edges, n_triplets, n_valid_triplets, n_kept_edges;
  uint32_t n_kept_views;
  uint32_t l1_iterations;            /* L1RA outer iterations run */
  uint32_t pd_iterations;            /* primal-dual Newton steps, over all L1RA iterations */
  uint32_t pd_backtracks;            /* rejected trial steps of the primal-dual line search, over all of them */
  uint32_t irls_iterations;
  int termination;                   /* of the last loop that ran (IRLS unless skipped): 0 it met the tolerance, 1 its
                                      * iteration cap, 2 a factorisation was not positive definite (the call returns the
                                      * rotations reached before it); -1 not run */
  double initial_l1_cost, final_l1_cost;  /* sum over kept edges of |log(R_j^T R_ij R_i)|_1 at the start and the end */
  double ms_triplets, ms_init, ms_l1, ms_irls, ms_device_total, ms_host;  /* ms_init: the host spanning tree */
} r3d_rotavg_l1_summary;
/* Replaces GlobalSfM_Rotation_AveragingSolver::Run with ROTATION_AVERAGING_L1 (OpenMVG 1.4, reached from
 * src/threads/R3DTriangulationThread.cpp:201-203 when Regard3D's rotation averaging method is "L1"): Chatterjee &
 * Govindu's robust rotation averaging.  Inputs, edge rules, triplet rejection, the kept component, error codes, the
 * R3D_ROTAVG_MAX_VIEWS limit, the gauge (the lowest kept view id gets R = I exactly) and the four outputs are those of
 * r3d_rotation_averaging; the solver on the kept component differs: a breadth-first spanning tree from the gauge view
 * (neighbours in ascending order) as the start, then L1RA (per iteration x = argmin |A x - b|_1, b_e = log(R_j^T R_ij
 * R_i), by l1-magic's primal-dual method, R_v <- R_v exp([x_v]x)), then IRLS with Geman-McClure weights.  Invalid
 * options: R3D_ERR_INVALID.  One global problem: it runs on the context's first device. */
int r3d_rotation_averaging_l1(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                              const r3d_rotavg_l1_options* opt, double* rotations, uint8_t* view_kept, uint8_t* edge_kept,
                              uint32_t* edge_support, r3d_rotavg_l1_summary* summary);
/* Diagnostics (device): one step of r3d_rotation_averaging_l1 through the members that function runs, on the same kept
 * component (m views, E edges, n = m - 1 free views).  kind 0: one Newton iteration of l1decode_pd (primal-dual), from
 * `state` at `tau` or, with state NULL, from the start point k_l1_pd_start forms at the residuals; then the rotations
 * updated by the resulting x, as after the last iteration of an L1RA step.  kind 1: one IRLS iteration.  kind 2: the
 * weighted normal equations (A^T diag(weights) A) dx = A^T rhs for n_systems (weights, rhs) pairs of 3E rows each, one
 * after the other on the same scratch.  A state is x (3n), A x, u, lambda_1, lambda_2 (3E each), A^T (lambda_1 -
 * lambda_2) (3n): 12 (E + n / 2) values.  Per-row arrays are E x 3 (row 3e + k), per-variable arrays component-major
 * (k n + a - 1).  Array outputs are caller-allocated for at most m = n_views and E = n_rel, NULL ones are skipped; the
 * scalars are always filled. */
typedef struct {
  uint32_t n_kept_views, n_kept_edges;  /* m, E; 0: no component, nothing else written */
  uint32_t* view_ids;       /* m: the kept view ids by local id (local 0: the gauge) */
  uint32_t* ab;             /* E x 2: each kept edge's local (a, b), a < b, in the kernels' order */
  double* Rk;               /* E x 9: its R_ab (R_b = R_ab R_a), row-major */
  double* rotations0;       /* m x 9: the rotations the step started from, by local id */
  double *b, *cost;         /* 3E, E: the residuals log(R_b^T R_ab R_a) there and |b_e|_1 */
  double bmax;              /* max |b| */
  int b_zero;               /* kind 0 from the start point: b = 0, so x = 0 and no iteration ran */
  /* kind 0 */
  double* state0;           /* the state the iteration started from */
  double sdg0, tau0, resnorm0;  /* its surrogate duality gap, tau and residual norm |(r_dual, r_cent)| */
  double *sigx, *rrow, *w2; /* 3E: the Newton system's row weights, right-hand-side rows and w2 */
  double* laplacians;       /* kinds 0, 1: 3 x (n + 1) x n, kind 2: n_systems of them: per component the Laplacian
                             * (rows 0..n-1) and the right-hand side A^T v (row n) as assembled, before factoring */
  int not_pd;               /* kinds 0, 1: the system was not positive definite (nothing after the solve ran) */
  double* dx;               /* kinds 0, 1: 3n; kind 2: n_systems x 3n, not written for a system that is not PD */
  double *Adx, *du, *dl1, *dl2;  /* 3E: the direction's other parts */
  double* Atdv;             /* 3n: A^T (dl1 - dl2) */
  double* rmin;             /* E: per edge min(1, its largest feasible step) */
  double step_max;          /* min over rmin: the ratio test's step before the 0.99 */
  uint32_t n_trials;        /* trial steps of the line search (<= 33) */
  double trial_step[33], trial_resnorm[33];  /* each trial's step and residual norm */
  int accepted;             /* the last trial was accepted (else the solver stops with the state it started from) */
  double* state;            /* the state after the iteration */
  double sdg, tau, resnorm; /* its values */
  /* kind 1 */
  double *w, *wb;           /* 3E: the Geman-McClure weights and w b */
  /* kinds 0, 1 */
  double* rotations;        /* m x 9: R_v exp([x_v]x) by local id (kind 0: x of the state after the iteration) */
  double xmax;              /* max |x| */
  /* kind 2 */
  int* sys_not_pd;          /* n_systems: each system was not positive definite */
} r3d_rotavg_l1_step_out;
/* rotations: NULL for the spanning-tree start, else n_views x 9 by view id (rotation_averaging_l1's layout; the kept
 * views' are read), finite.  kind 0: state NULL (n_state 0) or n_state = 12 E + 6 n finite values with u > |A x - b|
 * and lambda > 0 at the residuals, and tau > 0 finite; else R3D_ERR_INVALID.  kind 2: weights and rhs hold n_systems x
 * 3E values (n_systems >= 1).  opt: r3d_rotation_averaging_l1's (the kept component, irls_sigma_deg). */
int r3d_debug_rotavg_l1_step(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, uint32_t n_views,
                             const r3d_rotavg_l1_options* opt, const double* rotations, int kind, const double* state,
                             uint64_t n_state, double tau, const double* weights, const double* rhs, uint32_t n_systems,
                             r3d_rotavg_l1_step_out* out);
/* graph::CleanGraph_KeepLargestBiEdge_Nodes + KeepOnlyReferencedElement on a PairWiseMatches (how upstream's
 * GlobalSfMReconstructionEngine_RelativeMotions::Process() starts): the pairs whose views both lie in the largest
 * 2-edge-connected component of the pair graph (most views; a tie keeps the component holding the smallest view id).
 * Host only, like r3d_tracks_build. */
int r3d_matches_keep_largest_biedge_component(const r3d_matches* m, r3d_matches** out);

/* ---- global translations from the relative motions and the global rotations (global SfM, third step) ----------- */
#define R3D_TRANSAVG_L1 1            /* TRANSLATION_AVERAGING_L1 (the linear program): R3D_ERR_UNSUPPORTED here, solved by
                                      * r3d_translation_averaging_l1 */
#define R3D_TRANSAVG_L2_CHORDAL 2    /* TRANSLATION_AVERAGING_L2_DISTANCE_CHORDAL: 1DSfM chordal distance on the centres */
#define R3D_TRANSAVG_SOFTL1 3        /* TRANSLATION_AVERAGING_SOFTL1: soft-L1 on t_j - (R_ij t_i + s_ij t_ij), s_ij >= 1 */
/* The method values are Regard3D's transAveraging_ (src/threads/R3DTriangulationThread.cpp:204-208). */
typedef struct {
  int method;                        /* R3D_TRANSAVG_L2_CHORDAL (default) or R3D_TRANSAVG_SOFTL1 */
  double softl1_loss;                /* 0.01: SoftLOneLoss width of R3D_TRANSAVG_SOFTL1 */
  r3d_ba_options lm;                 /* the trust region.  Honoured: gradient_tolerance, parameter_tolerance,
                                      * initial_radius; max_iterations if > 0 (0: the method's cap, 500 for chordal,
                                      * max(50, 2 x kept edges) for soft-L1); function_tolerance if > 0 (0: 1e-7 for
                                      * chordal, 1e-6 for soft-L1).  huber_a, refine_intrinsics, prior_huber_a unused. */
} r3d_transavg_options;
void r3d_transavg_default_options(r3d_transavg_options* o);  /* L2 chordal, 0.01, the methods' upstream tolerances */
typedef struct {
  int success;                       /* 0: no bi-edge-connected component among the usable edges */
  uint64_t n_edges;                  /* usable entries: OK, edge_use set, both views rotation-kept */
  uint64_t n_kept_edges;
  uint32_t n_kept_views;
  uint32_t lm_iterations, lm_successful_steps;
  int lm_termination;                /* as r3d_ba_summary.termination; -1: not run */
  double lm_initial_cost, lm_final_cost;
  double ms_solve, ms_device_total, ms_host;
} r3d_transavg_summary;
/* Replaces GlobalSfMReconstructionEngine_RelativeMotions::Compute_Global_Translations (OpenMVG 1.4, reached from
 * src/threads/R3DTriangulationThread.cpp:201-250) for the chordal and soft-L1 methods, with the pairwise relative
 * translations of r3d_relative_poses in place of upstream's triplet-wise ones (DESIGN.md sec. 2).  Edges: the OK entries
 * of rel whose edge_use is set (NULL: every OK entry; pass rotation averaging's edge_kept) and whose views are both in
 * rot_kept; the largest bi-edge-connected component of them.  rotations: n_views x 9 from r3d_rotation_averaging.
 *   chordal: unknown centres C, one residual (C_J - C_I) / |C_J - C_I| + R_J^T t_IJ / |t_IJ| per edge, no loss, start
 *            from a fixed pseudo-random draw in [0, 1).
 *   soft-L1: unknown translations t and one scale s >= 1 per edge, residual t_J - (R_J R_I^T t_I + s t_IJ / |t_IJ|),
 *            SoftLOneLoss(softl1_loss), start t = 1, s = 1.
 * Gauge: the lowest kept view id gets C = 0 (chordal) / t = 0 (soft-L1) exactly and is held.  Outputs: centers and
 * translations n_views x 3 (t = -R C; zero for views outside the component), view_kept n_views, edge_kept n_rel (may be
 * NULL).  I == J, a view id >= n_views, an unordered pair given twice or a zero / non-finite translation among the OK
 * entries with edge_use set: R3D_ERR_INVALID; more than R3D_ROTAVG_MAX_VIEWS kept views or method L1:
 * R3D_ERR_UNSUPPORTED.  One global problem: it runs on the context's first device. */
int r3d_translation_averaging(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                              const double* rotations, const uint8_t* rot_kept, uint32_t n_views,
                              const r3d_transavg_options* opt, double* centers, double* translations, uint8_t* view_kept,
                              uint8_t* edge_kept, r3d_transavg_summary* summary);

/* ---- global translations by Regard3D's default method, TRANSLATION_AVERAGING_L1 ----------------------------------- */
typedef struct {
  int max_iterations;                /* 100: interior-point iterations (>= 1) */
  double tolerance;                  /* 1e-9: stop when max |G y + s - h| <= tol (1 + |h|_inf), max |G^T z + c| <= tol and
                                      * |gamma - dual objective| <= tol (1 + |gamma|) (> 0) */
} r3d_transavg_l1_options;
void r3d_transavg_l1_default_options(r3d_transavg_l1_options* o);  /* 100, 1e-9 */
typedef struct {
  int success;                       /* as r3d_transavg_summary */
  uint64_t n_edges, n_kept_edges;
  uint32_t n_kept_views;
  uint32_t iterations;               /* predictor-corrector iterations */
  uint32_t regularized_factorizations;  /* retries of a factorisation that was not positive definite, each with
                                      * 1e-18, 1e-16, ... (x 100, at most 5) times the largest diagonal entry added */
  int termination;                   /* 0 converged, 1 iteration cap, 2 factorisation failed, -1 not run */
  double gamma;                      /* the L-infinity bound of the returned point (the LP's objective) */
  double dual_objective;
  double max_primal_violation;       /* largest violation of a constraint by the returned point (>= 0) */
  double max_dual_violation;         /* max |G^T z + c| */
  double ms_solve, ms_device_total, ms_host;
} r3d_transavg_l1_summary;
/* Replaces GlobalSfM_Translation_AveragingSolver::Translation_averaging for TRANSLATION_AVERAGING_L1 (OpenMVG 1.4,
 * Tifromtij_ConstraintBuilder + the CLP solver; Regard3D's default, src/threads/R3DTriangulationThread.cpp:204): the
 * L-infinity translation registration of Moulon et al. (ICCV 2013) on the pairwise relative translations, one scale per
 * edge:  minimise gamma  s.t.  |(T_J - R_J R_I^T T_I - lambda_IJ t_IJ / |t_IJ|)_k| <= gamma,  lambda_IJ >= 1, by a
 * primal-dual interior-point method (Mehrotra predictor-corrector) on the first device.  Inputs, edge rules, the kept
 * component, the gauge (the lowest kept view id gets T = 0) and the outputs centers / translations / view_kept /
 * edge_kept as r3d_translation_averaging's soft-L1 method; edge_scale (n_rel, may be NULL): lambda of the kept edges,
 * 0 elsewhere.  The optimal value gamma is unique, the optimal point in general is not: the method returns a point near
 * the centre of the optimal face, not a vertex.  Errors as r3d_translation_averaging, and R3D_ERR_INVALID for
 * max_iterations < 1 or tolerance <= 0. */
int r3d_translation_averaging_l1(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                                 const double* rotations, const uint8_t* rot_kept, uint32_t n_views,
                                 const r3d_transavg_l1_options* opt, double* centers, double* translations, uint8_t* view_kept,
                                 uint8_t* edge_kept, double* edge_scale, r3d_transavg_l1_summary* summary);

/* ---- the steps either side of bundle adjustment (SURVEY.md 8f-3) -------------------------------------------------
 * openMVG::tracks::TracksBuilder Build + Filter(min_length) + ExportToSTL, as Regard3D calls them itself
 * (src/threads/PreviewGeneratorThread.cpp:345-352) and as every SfM engine it drives starts: union-find over the
 * pairwise matches; tracks with two features of one image or fewer than min_length images are dropped.  Tracks come
 * in track-id order (upstream: the union-find root), each as its (view, feature) pairs in view order. */
typedef struct r3d_tracks r3d_tracks;
int r3d_tracks_build(const r3d_matches* m, uint32_t min_length /* 2 */, r3d_tracks** out);
uint64_t r3d_tracks_count(const r3d_tracks* t);
int r3d_tracks_get(const r3d_tracks* t, uint64_t k, uint32_t* track_id, const uint32_t** views, const uint32_t** feats,
                   uint32_t* n);
/* TracksUtilsMap::GetTracksInImages (PreviewGeneratorThread.cpp:354-358): tracks seen in ALL listed views, cut to them */
int r3d_tracks_in_images(const r3d_tracks* t, const uint32_t* view_ids, uint32_t n, r3d_tracks** out);
void r3d_tracks_free(r3d_tracks* t);
/* Tracks -> sd.structure (observation = position of the feature, from r3d_upload_regions of that view id), then
 * SfM_Data_Structure_Computation_Blind::triangulate: every landmark from all its views with a pose and an intrinsic
 * (iteratively re-weighted DLT); landmarks with fewer than two such views or a non-positive depth are erased. */
int r3d_sfm_structure_from_tracks(r3d_ctx* ctx, r3d_sfm_data* sd, const r3d_tracks* tracks, uint32_t* n_rejected);
/* RemoveOutliers_PixelResidualError(sd, max_pixel_residual, min_track_length) then RemoveOutliers_AngleError(sd,
 * min_angle_deg) -- the rejection step the engines run after each bundle adjustment (4.0 px / 2.0 degrees upstream).
 * min_angle_deg <= 0 skips the angle test. */
int r3d_sfm_remove_outliers(r3d_ctx* ctx, r3d_sfm_data* sd, double max_pixel_residual, uint32_t min_track_length,
                            double min_angle_deg, uint32_t* removed_observations, uint32_t* removed_landmarks);

/* ---- after the engine: the coloured model and the undistorted views (DESIGN.md 4.5i) -------------------------------
 * The plan of OpenMVGHelper::ColorizeTracks (src/utils/OpenMVGHelper.cpp:2453-2560), the greedy loop the triangulation
 * step runs after Process() (src/threads/R3DTriangulationThread.cpp:461-476, :267-278): each round counts, per view, the
 * observations of the landmarks not coloured yet, picks the first view in id order with the largest count
 * (sort_index_helper with nbuplet = 1: std::partial_sort under val >, a first-max), and every remaining landmark that
 * view observes takes its colour from that view's image at (int)y, (int)x (truncated toward zero).  The whole loop runs
 * on the device; the images stay with the caller, who reads them in round_view order and gathers rgb[y][x].
 * round_view: num_views entries, the view id chosen in each of the *n_rounds rounds; lm_round: per landmark in id order,
 * the round that colours it; lm_pixel: per landmark, (x, y) in that round's image.  R3D_ERR_INVALID before any device
 * work for: a landmark without observations, an observation whose truncated position lies outside its view's
 * width x height, an observation of a view without a pose or intrinsic (never in a reconstructed scene).  A pose shared by
 * views with different intrinsics: R3D_ERR_UNSUPPORTED (the scene as r3d_sfm_bundle_adjust reads it).  Runs on the
 * context's first device. */
int r3d_sfm_colorize_plan(r3d_ctx* ctx, const r3d_sfm_data* sd, uint32_t* round_view, uint32_t* n_rounds,
                          uint32_t* lm_round, int32_t* lm_pixel);
/* Host only: FinalColorized.ply as plyHelper::exportToPly writes it with colours (SfMPlyHelper.hpp:62-116): an ASCII
 * header, every landmark in id order as "x y z r g b" (std::fixed, precision 16; colors: num_landmarks x 3 in landmark
 * id order, NULL = 255 255 255), then the centre of every pose in pose-id order with 0 255 0.  R3D_ERR_IO naming the
 * path. */
int r3d_sfm_write_colorized_ply(const r3d_sfm_data* sd, const uint8_t* colors, const char* path);

/* OpenMVG 1.4's UndistortImage(image, cam, image_ud, BLACK), which every densification export runs on every
 * reconstructed view (OpenMVGHelper.cpp:750, :1223, :1377, :1819, :2093, :2281, :2860, :3026,
 * OpenMVGExportToMVS.cpp:157).  Per view: a pinhole intrinsic copies the image; every other model (zero coefficients
 * too) fills black, then each output pixel (i, j) whose distorted position d = cam2ima(add_disto(ima2cam(i, j)))
 * (double) satisfies Contains((int)d.y, (int)d.x) takes Sampler2d<SamplerLinear>(in, (float)d.y, (float)d.x): float
 * weights over the 2 x 2 taps from floor, taps outside the image dropped, the sum accumulated in double and divided by
 * the total weight when that is not 1, total weight <= 0.2: black; the value clamped to [0, 255] and truncated
 * (DESIGN.md 2.4).  rgb[k] / out[k]: heights[k] x widths[k] x 3 uint8, row-major; intr[k]: the view's intrinsic (its
 * model, focal, principal point and disto; its width / height are not read).  R3D_ERR_INVALID before any work for a
 * NULL pointer, a zero width or height, an unknown model.  Images are dealt to the context's devices in contiguous
 * runs; on each, pinned staging buffers double-buffer the uploads (copy stream) against the kernel and downloads
 * (compute stream).  timing (may be NULL): the call's stage times. */
typedef struct {
  double upload_ms;    /* host -> device copies (CUDA events, summed over images and devices) */
  double kernel_ms;    /* the undistortion kernels */
  double download_ms;  /* device -> host copies */
  double stage_ms;     /* host copies into and out of the pinned staging buffers (wall time, summed over devices) */
  double total_ms;     /* the call's wall time */
  uint32_t images, copied, kernel_launches, devices;  /* copied: pinhole views */
} r3d_undistort_timing;
int r3d_undistort_images(r3d_ctx* ctx, uint32_t n, const r3d_sfm_intrinsic* intr, const uint8_t* const* rgb,
                         const uint32_t* widths, const uint32_t* heights, uint8_t* const* out, r3d_undistort_timing* timing);

/* ---- multi-GPU bundle adjustment (SURVEY.md 8e: the one path with a real exchange step) -------
 * One process per GPU.  The 3-D points (with all their observations) are partitioned over the
 * ranks, cameras and intrinsics are replicated: every rank passes r3d_bundle_adjust ALL cameras /
 * intrinsics and ITS points + observations.  Per LM iteration the partial reduced camera system
 * S = U - sum W V^-1 W^T and its right-hand side are summed over the ranks with ONE ncclAllReduce
 * (double) over NVLink, the dense Cholesky is replicated, back-substitution is local; cost, camera
 * gradient / Jacobi scaling and the step norms are small all-reduces.  On return poses/intrinsics
 * are identical on every rank, points hold the rank's own slice.  There is no reference counterpart
 * (Ceres is single-process); parity is against the single-GPU path / the oracle.
 * libnccl.so.2 is resolved at run time (the copy already loaded in the process, e.g. torch's, else
 * $R3D_NCCL_LIB, else the system one).  The id is created on rank 0 and distributed by the host
 * (torch.distributed / MPI / a file). */
#define R3D_COMM_ID_BYTES 128
int r3d_comm_unique_id(r3d_ctx* ctx, uint8_t id[R3D_COMM_ID_BYTES]);
int r3d_comm_init(r3d_ctx* ctx, int world, int rank, const uint8_t id[R3D_COMM_ID_BYTES]);
int r3d_comm_destroy(r3d_ctx* ctx);
int r3d_comm_world(const r3d_ctx* ctx);   /* 1 when no communicator is attached */
/* OpenMVGHelper::calculateResiduals (src/utils/OpenMVGHelper.cpp:2572-2590): |residual| per
 * coordinate, 2 per observation -- the BA quality metric the GUI reports. */
int r3d_ba_residuals(r3d_ctx* ctx, const r3d_ba_problem* p, double* res /* n_obs x 2 */);

/* ---- file-level twin of R3DComputeMatches::computeMatches() --------------------------------- */
#define R3D_MATCHING_CASCADE_HASHING 100 /* not a value of the reference's matchingAlgorithm switch */
typedef void (*r3d_progress_cb)(float fraction, const char* message, void* user);

typedef struct {
  float dist_ratio;               /* R3DFParams::distRatio_ (src/Regard3DFeatures.h:52-69) */
  int compute_fundamental;        /* R3DFParams::computeFundalmentalMatrix_ */
  int compute_essential;          /* R3DFParams::computeEssentialMatrix_ -> matches.e.txt (+ the poor-overlap filter) */
  int compute_homography;         /* R3DFParams::computeHomographyMatrix_ -> matches.h.txt */
  int matching_algorithm;         /* 0..8 as src/R3DComputeMatches.cpp:2036-2062; all map to the exact GPU matcher.
                                   * Extension: R3D_MATCHING_CASCADE_HASHING selects R3D_MATCH_CASCADE_HASHING */
  uint32_t descriptor_dim;        /* 144 for R3D_AKAZE_LIOP_Regions */
  int svg_output;                 /* computeMatches(..., bool svgOutput, ...): PutativeAdjacencyMatrix.svg and
                                   * GeometricAdjacencyMatrix.svg in the matches dir (:2074-2076, :2238-2240) */
} r3d_cm_params;

typedef struct {
  const char* matches_dir;        /* R3DProjectPaths::relativeMatchesPath_ : holds <img>.feat/.desc, outputs */
  const char* const* image_basenames; /* n_views names without extension (image%06d, src/R3DProject.cpp:1042) */
  const r3d_view_info* views;     /* image sizes (sfm_data views) */
  uint32_t n_views;
  const char* matches_f_filename; /* R3DProjectPaths::matchesFFilename_ ; NULL -> <matches_dir>/matches.f.txt */
  const char* matches_h_filename; /* R3DProjectPaths::matchesHFilename_ ; NULL -> <matches_dir>/matches.h.txt */
  const char* matches_e_filename; /* R3DProjectPaths::matchesEFilename_ ; NULL -> <matches_dir>/matches.e.txt */
} r3d_cm_paths;

typedef struct {
  uint32_t n_views;
  uint32_t* number_of_keypoints;  /* caller array of n_views (R3DComputeMatchesStatistics::numberOfKeypoints_) */
  uint64_t putative_pairs, putative_matches, f_pairs, f_matches, h_pairs, h_matches, e_pairs, e_matches;
  double seconds_load, seconds_match, seconds_filter;
} r3d_cm_stats;

/* Steps of R3DComputeMatches::computeMatches() after feature extraction
 * (src/R3DComputeMatches.cpp:2035-2126): load regions, exhaustive pairs, putative matching,
 * Save(matches.putative.txt), F filter, Save(matches.f.txt), E filter + poor-overlap removal (< 50 inliers or
 * < 30 % of the putatives, :2173-2191), Save(matches.e.txt), H filter, Save(matches.h.txt); progress fractions
 * as the reference emits them (0.7 putative, 0.8 F, 0.9 E, 0.95 H; SURVEY.md sec. 5). */
int r3d_compute_matches(r3d_ctx* ctx, const r3d_cm_params* params, const r3d_cm_paths* paths,
                        r3d_progress_cb cb, void* user, r3d_cm_stats* stats);

/* ---- instrumentation ----------------------------------------------------------------------- */
typedef struct {
  double ms_prep;        /* upload-time operand preparation kernels */
  double ms_candidates;  /* wgmma candidate kernel(s), CUDA-event time on their stream */
  double ms_rerank;      /* exact re-rank + ratio kernel(s) */
  double ms_fallback;    /* exact-scan kernel for uncertified queries + the per-pair pack / (i,j) sort kernel */
  double ms_device_total;/* first launch -> last kernel of the last r3d_match_pairs */
  double ms_host_post;   /* host de-duplication */
  uint64_t kernel_launches;
  uint64_t queries, fallback_queries, third_chunk_queries, fifth_chunk_queries;  /* R3D_MATCH_CASCADE_HASHING: the last two count
                                                                                 * raw / distinct bucket candidates instead */
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t rejected_queries; /* dropped before any exact distance: the ratio test provably cannot pass */
} r3d_match_timing;
int r3d_get_match_timing(const r3d_ctx* ctx, r3d_match_timing* out);

typedef struct {
  double ms_solve, ms_score, ms_device_total, ms_host;
  uint64_t kernel_launches, hypotheses, rounds;
} r3d_filter_timing;
int r3d_get_filter_timing(const r3d_ctx* ctx, r3d_filter_timing* out);

/* Diagnostics (host only, no GPU needed): IndMatch::getDeduplicated + IndMatchDecorator::getDeduplicated of one
 * pair, in place; returns the new count.  The CPU test pins it against std::set. */
int64_t r3d_debug_post_process(r3d_indmatch* m, int64_t n, const float* xyI, const float* xyJ, int coord_dedup);
/* the same for up to 4 pairs advanced in lockstep by one thread (what the batch tails call) */
int r3d_debug_post_process_many(int lanes, r3d_indmatch* const* ms, uint64_t* counts, const float* const* xyIs,
                                const float* const* xyJs, int coord_dedup);
/* the descent-free replay the batch tails use (per-view y-rank / shared-x tables, built here from the n_keypoints
 * positions of view I) */
int64_t r3d_debug_post_process_ranked(r3d_indmatch* m, int64_t n, const float* xyI, uint32_t n_keypoints, const float* xyJ);

/* Diagnostics (host only): 1 when the library's device-side restatement of std::mt19937 +
 * std::uniform_int_distribution<uint32_t> (the ACRANSAC sample stream) reproduces this process's <random>.  When it
 * does not (another standard library), r3d_filter_pairs, r3d_relative_poses and r3d_resect_views return
 * R3D_ERR_UNSUPPORTED. */
int r3d_debug_rng_selftest(void);
/* Diagnostics (device): the AC-RANSAC kernel's scoring of caller-supplied models on one pair, through the device code
 * the F / H / E filters, r3d_relative_poses and r3d_resect_views run.  model: internal id 0 = F (symmetric epipolar
 * error, 9 doubles), 1 = H (asymmetric transfer error, 9), 2 = E as F = K2^-T E K1^-1 (one-sided epipolar distance in
 * pixels, 9), 3 = resection (reprojection error of P = K [R | t], 12 doubles, row-major 3 x 4).  x1, x2: M x 2
 * (model 3: x1 = X.xy, x2 = the pixel), x3: X.z (model 3 only, NULL otherwise), M >= the model's minimal sample.
 * max_thr: the squared precision bound (+inf only for model 3); K[6]: the pair's AcPair.K (model 3: K[3] > 0 is where
 * the tier-1 histogram's top bin starts).  loge0 and the float log-combination tables are built as the filters build
 * them; the size class (shared-memory or global sort) is the one the filters would pick for M.
 * Per model, out[m]: lb = the tier-1 lower bound of the best NFA, cnt_hi / cnt_lo = the tier-1 upper / lower count of
 * the residuals <= max_thr, count = their exact number, nfa / k / err = the tier-2 best NFA, its number of inliers and
 * the k-th smallest residual.  Optional (may be NULL): lo / hi / e, n_models x M, the tier-1 interval and the tier-2
 * residual of every (model, point); logc_n (M + 2: log10 C(M, k) for k = 0 .. M, then the table's error bound) and
 * logc_k (M + 1). */
typedef struct {
  double lb, nfa, err;
  uint32_t cnt_hi, cnt_lo, count, k;
} r3d_ac_score;
int r3d_debug_acransac_score(r3d_ctx* ctx, int model, uint32_t M, const double* x1, const double* x2, const double* x3,
                             double max_thr, double logalpha0, const double* K, const double* models, uint32_t n_models,
                             r3d_ac_score* out, double* lo, double* hi, double* e, float* logc_n, float* logc_k);
/* Diagnostics: the library's deterministic transcendental functions (detmath.cuh) on n inputs, on the current CUDA
 * device (on_device != 0) or in the library's host code.  fn: 0 = log10, 1 = cbrt, 2 = cos, 3 = acos. */
int r3d_debug_detmath(int fn, int on_device, const double* x, uint64_t n, double* y);
/* test hook: hash tables of a prepared view (code n x ceil(dim/32), bucket n x 6, bk_ofs 6 x 1025, bk_ids 6 x n) */
int r3d_debug_cascade_view(r3d_ctx* ctx, uint32_t view_id, uint32_t* code, uint16_t* bucket, uint32_t* bk_ofs, uint32_t* bk_ids);

/* Diagnostics: the packed candidate keys per query row (n_query padded to 256 rows x 8 uint32:
 * 6 keys ascending + 2 unused)
 * the tensor-core pass produced for (view_db, view_query), and the pair's error bound. */
int r3d_debug_candidate_keys(r3d_ctx* ctx, uint32_t view_db, uint32_t view_query, uint32_t* keys,
                             float* eps_abs);
/* Diagnostics: the fp16 tensor-core operands of one view, prepared as the next matching call prepares them (every
 * uploaded view of the first device).  *n_pad: padded rows; *kp: halves per operand row, 0 when the view has no fp16
 * operands (integer path or exact scan only).  opQ / opD (may be NULL): n_pad x kp fp16 bit patterns of the query and
 * database roles; stats (may be NULL): max ||a||^2, max ||fp16(a)||^2, max ||a - fp16(a)||^2, max |a_k| over the rows;
 * *e0 (may be NULL): the norm-split exponent of the device (S0 = 2^e0, S1 = 2^(e0-11)). */
int r3d_debug_view_operands(r3d_ctx* ctx, uint32_t view_id, uint32_t* n_pad, uint32_t* kp, uint16_t* opQ, uint16_t* opD,
                            float* stats, int* e0);

/* Diagnostics (runs on the host, no GPU needed): residual and analytic Jacobian (2 x 15: intrinsics
 * 0..5, pose 6..11, point 12..14) of one observation, as the BA kernels evaluate them. */
int r3d_debug_ba_jacobian(const double* intr, const double* pose, const double* X, const double* obs,
                          double* r, double* J);
/* the same for any of the five camera models (ext: the model's coefficients 4, 5 or NULL) */
int r3d_debug_ba_jacobian_model(int model, const double* intr, const double* ext, const double* pose, const double* X,
                                const double* obs, double* r, double* J);
/* pose-centre prior block: r[3] = weight .* (C(pose) - center), J[3 x 6] = d r / d (angle-axis, t) */
int r3d_debug_ba_prior(const double* pose, const double* center, const double* weight, double* r, double* J);

/* Diagnostics (device): the library's dense solvers on a caller's matrix, through the launch code the solvers use.
 * Factor A = L L^T and solve A x = b.  A is (n+1) x n row-major: rows 0..n-1 the matrix (only the lower triangle is
 * read), row n the right-hand side b.  method 0 = k_chol_fused, the cooperative kernel of bundle adjustment, rotation
 * and translation averaging (grid = CTAs, 0 = one per SM as those solvers launch it); method 1 = k_chol_envelope, the
 * envelope kernel of R3D_BA_CHOL=envelope (n even; ft = first column tile of each of the ceil((n+1)/32) row tiles,
 * 0 <= ft[t] <= t, at most 24 active row tiles per panel; grid = cluster size 1..8, 0 = 8).  Outputs: L_out (n+1) x n
 * (the factor, zero above the diagonal; row n = y = L^-1 b), x_out (n) = A^-1 b, Linv_out (method 0 only, may be NULL:
 * ceil(n/32) row-major 32 x 32 inverses of the diagonal blocks of L, identity-padded), *not_pd = 1 when the
 * factorisation met a pivot that is not > 0 (or NaN).  Bad arguments return R3D_ERR_INVALID before anything runs. */
int r3d_debug_cholesky(r3d_ctx* ctx, int method, int n, const double* A, const int* ft, int grid, double* L_out,
                       double* x_out, double* Linv_out, int* not_pd);
/* A X = Y for 3 right-hand sides: k_chol_fused as rotation averaging launches it, then k_rotavg_trsm3 exactly as one
 * inverse iteration of its initialisation runs it.  A n x n row-major (lower triangle read), Y and X_out n x 3
 * row-major; grid = CTAs of the triangular solves, 0 = the occupancy the initialisation uses.  R3D_ERR_INVALID when
 * A is not positive definite. */
int r3d_debug_chol_solve3(r3d_ctx* ctx, int n, const double* A, const double* Y, int grid, double* X_out);

/* Diagnostics (device): one bundle-adjustment LM step at the problem's parameters, through the code r3d_bundle_adjust
 * runs per iteration, with the Jacobi scaling made at those parameters.  nB = 6 n_cams (+ 6 n_intr when
 * refine_intrinsics), nparam = nB + 3 n_pts; parameter order: poses, intrinsic groups, points.  Array outputs are
 * caller-allocated, NULL ones are skipped; the scalars are always filled. */
typedef struct {
  double* g;        /* nparam: scaled gradient J^T r (Huber-corrected, Jacobi-scaled) */
  double* diag;     /* nparam: scaled diag(J^T J) */
  double* scale;    /* nparam: Jacobi scaling 1 / (1 + |column|) */
  double* S;        /* nB x nB: the reduced camera system, both triangles, with D^2 = clamp(diag, 1e-6, 1e32) / radius */
  double* rhs;      /* nB: its right-hand side */
  double* Vinv;     /* n_pts x 9: (sum Jp^T Jp + D^2)^-1 per point */
  double* delta;    /* nparam: the step (scaled coordinates) */
  uint32_t nB, n_batches, n_long;  /* the batched Schur kernel's CTAs, the points of the CTA-per-point kernel */
  int not_pd;       /* the Cholesky met a pivot that is not > 0 */
  double gmax, model_cost_change, dx_norm2, x_norm2;  /* max |unscaled g|, model cost change, |dx|^2, |x|^2 */
} r3d_ba_step_out;
/* schur_route 0 = the default plan (batched kernel where it applies), 1 = every point through the CTA-per-point kernel
 * (as R3D_BA_SCHUR=point); chol_method 0 = dense, 1 = envelope (R3D_ERR_INVALID where that kernel does not apply).
 * Uses opt->huber_a, refine_intrinsics and prior_huber_a. */
int r3d_debug_ba_step(r3d_ctx* ctx, const r3d_ba_problem* p, const r3d_ba_options* opt, double radius, int schur_route,
                      int chol_method, r3d_ba_step_out* out);

/* Diagnostics (device): one predictor-corrector iteration of r3d_translation_averaging_l1, through the code that
 * function runs per iteration, on the same kept edges.  A state is packed as y (N = 3 (m - 1) + 1: T of the free kept
 * views in local order, then gamma), lambda (ne), s (7 ne), z (7 ne), the last three in kept-edge order and the 7 rows
 * of an edge as the LP's (r_k - gamma, -r_k - gamma for k = 0..2, -lambda).  Array outputs are caller-allocated for at
 * most m = n_views kept views and ne = n_rel kept edges, NULL ones are skipped; the scalars are always filled. */
typedef struct {
  uint32_t n_kept_views, n_kept_edges, n;  /* m, ne, N; 0: no component, nothing else written */
  uint32_t* view_ids;       /* m: the kept view ids by local id (local 0: the gauge) */
  uint64_t* edge_record;    /* ne: each kept edge's record */
  uint32_t* edge_ij;        /* ne x 2: its record-oriented local (I, J) */
  double* Rij;              /* ne x 9: R_J R_I^T (row-major) as the kernels use it */
  double* u;                /* ne x 3: t_IJ / |t_IJ| as the kernels use it */
  double* state0;           /* N + 15 ne: the state the iteration started from */
  double norms[5];          /* k_tl_norms: max |G y + s - h|, max(0, G y - h), max |G^T z + c|, s^T z, -h^T z */
  double* A;                /* (N + 1) x N: the reduced (T, gamma) system as assembled, before scaling (rows 0..N-1;
                             * the T block in full, the gamma row N - 1, the gamma column above it not written: 0),
                             * row N: the predictor's right-hand side */
  double* sc;               /* N: the Jacobi scale, 1 / sqrt(A_ii) (1 where A_ii <= 0) */
  int not_pd[6];            /* per factorisation attempt of the predictor: it met a pivot that is not > 0 */
  uint32_t retries;         /* attempts after the first (each with the diagonal raised) */
  double *pred_dy, *pred_dlam, *pred_ds, *pred_dz;  /* N, ne, 7 ne, 7 ne: the predictor's step (dy refined, unscaled) */
  double pred_alpha_p, pred_alpha_d, pred_complementarity;  /* its step lengths (eta = 1), (s + a_p ds)^T (z + a_d dz) */
  double sigma;             /* the centring (mu_aff / mu)^3 */
  double* corr_rhs;         /* N: the corrector's right-hand side, scaled by sc */
  double *corr_dy, *corr_dlam, *corr_ds, *corr_dz;  /* the corrector's step */
  double alpha_p, alpha_d;  /* its step lengths (eta = 0.99) */
  double* state;            /* N + 15 ne: the state after the step */
  int converged;            /* the stopping test held at the start: nothing after the norms and A ran */
  int failed;               /* every factorisation attempt failed: nothing after the predictor ran */
} r3d_transavg_l1_step_out;
/* state: NULL for the solver's start point, else N + 15 ne values (n_state), finite, s > 0 and z >= 0, or
 * R3D_ERR_INVALID.  tolerance: the stopping test's (r3d_transavg_l1_options). */
int r3d_debug_transavg_l1_step(r3d_ctx* ctx, const r3d_relative_pose* rel, uint64_t n_rel, const uint8_t* edge_use,
                               const double* rotations, const uint8_t* rot_kept, uint32_t n_views, const double* state,
                               uint64_t n_state, double tolerance, r3d_transavg_l1_step_out* out);

/* ---- keypoints (SURVEY.md 3: the feature stage's detector) ------------------------------------------------------ */
/* Two of Regard3DFeatures::detectKeypoints' detectors on one scale space:
 *   R3D_DETECTOR_FAST_AKAZE  the "Fast-AKAZE" branch (src/Regard3DFeatures.cpp:590-614) with cv::AKAZE2 of
 *                            src/thirdparty/fast-akaze; the default of R3DFParams (:133)
 *   R3D_DETECTOR_AKAZE       the "AKAZE" branch (:578-589): OpenCV 4's cv::AKAZE::detect; the compute-matches
 *                            dialog's default (keyPointDetectorType_ 0), which is what a default GUI run uses
 * Input: float gray images in [0, 1] as R3DFeaturesThread::processWorkItem builds them
 * (src/threads/R3DFeaturesThread.cpp:162-191); decoding stays with the caller.  PM_G2 is the only diffusivity the
 * detectors implement. */
#define R3D_DETECTOR_FAST_AKAZE 0
#define R3D_DETECTOR_AKAZE 1
#define R3D_AKAZE_DIFF_PM_G2 1 /* KAZE::DIFF_PM_G2 */
typedef struct {
  float threshold;     /* detector response threshold (R3DFParams::threshold_, default 0.001) */
  int32_t octaves;     /* 4 */
  int32_t sublevels;   /* 4 */
  int32_t diffusivity; /* R3D_AKAZE_DIFF_PM_G2 */
} r3d_akaze_options;
void r3d_akaze_default_options(r3d_akaze_options* out);

/* cv::KeyPoint as the detector leaves it, in upstream order (levels ascending, then each level's candidate order,
 * which is raster order for AKAZE): size = diameter, class_id = evolution level.  angle, in degrees: Fast-AKAZE's after
 * Regard3D's conversion (radians * 180 / pi + 90, wrapped into [0, 360]); AKAZE's as cv::AKAZE returns it
 * (fastAtan2, [0, 360), no conversion), which is what Regard3D passes on for that detector. */
typedef struct {
  float x, y, size, angle, response;
  int32_t octave, class_id;
} r3d_akaze_keypoint;

/* one evolution level of an image of the given size: (octave, sublevel), its shape, derivative kernel scale, border,
 * sigma, diffusion time, octave ratio and the number of FED steps that lead to it from the previous level */
typedef struct {
  int32_t octave, sublevel, width, height, sigma_size, border;
  float esigma, etime, ratio;
  uint32_t n_tau;
} r3d_akaze_level;
/* the level table of a width x height image; returns the number of levels (at most cap are written) or < 0 */
int r3d_akaze_levels(uint32_t width, uint32_t height, const r3d_akaze_options* opt, r3d_akaze_level* out, int cap);

/* Keypoints of a batch of images (opaque, host memory). */
typedef struct r3d_features r3d_features;
/* images[i]: width[i] x height[i] row-major float32.  R3D_ERR_INVALID before any work for a side <= 2, a non-finite
 * pixel or a bad option.  The images are dealt to the context's devices in contiguous slices and processed there in
 * batches bounded by the device memory; the result does not depend on the number of devices.  An image too small for
 * the first level (2 border + 1 >= a side, border 29 at the defaults) has no keypoints: upstream asserts instead. */
int r3d_akaze_detect(r3d_ctx* ctx, const float* const* images, const uint32_t* widths, const uint32_t* heights,
                     uint32_t n_images, const r3d_akaze_options* opt, r3d_features** out);
/* r3d_akaze_detect with a choice of detector (R3D_DETECTOR_*; r3d_akaze_detect is R3D_DETECTOR_FAST_AKAZE).  The same
 * inputs are rejected, and an unknown detector is R3D_ERR_INVALID.  Both detectors share the scale space, the
 * candidates (3x3 maxima above the threshold inside the border) and the orientation search; they differ in the
 * extrema passes and in where a refined point is placed (DESIGN.md 2.3). */
int r3d_detect_keypoints(r3d_ctx* ctx, int detector, const float* const* images, const uint32_t* widths,
                         const uint32_t* heights, uint32_t n_images, const r3d_akaze_options* opt, r3d_features** out);
uint32_t r3d_features_num_images(const r3d_features* f);
uint32_t r3d_features_count(const r3d_features* f, uint32_t image);
const r3d_akaze_keypoint* r3d_features_get(const r3d_features* f, uint32_t image);
void r3d_free_features(r3d_features* f);

/* per-stage device time of the last r3d_akaze_detect (CUDA events, milliseconds, summed over batches and devices) */
typedef struct {
  double upload_ms;        /* images host -> device, workspace clears */
  double scale_space_ms;   /* blur, Scharr, k-percentile, Hessian, conductivity, FED */
  double candidates_ms;    /* 3x3 maxima and their raster-order compaction */
  double same_level_ms;    /* the same-level pass alone */
  double cross_level_ms;   /* the lower- and the upper-level pass */
  double refine_orient_ms; /* subpixel refinement, orientation, copies back */
  double total_ms;
  uint32_t images, batches, keypoints, kernel_launches, devices;
} r3d_akaze_timing;
int r3d_get_akaze_timing(const r3d_ctx* ctx, r3d_akaze_timing* out);

/* Diagnostics: one image through r3d_akaze_detect's kernels, every level kept.  arrays: per level, in level order,
 * Lt, Lsmooth, Lx, Ly, Ldet (5 x width x height floats each); kcontrast: per level (0 for a single-level image);
 * cands / flags: per level, in level order, the candidates after the same-level pass (angle -1) and their deletion
 * flags (bit 0: by the lower-level pass, bit 1: after the upper-level pass); cand_counts: per level.  Returns
 * R3D_ERR_INVALID when more than cand_cap candidates exist. */
int r3d_debug_akaze_levels(r3d_ctx* ctx, const float* image, uint32_t width, uint32_t height, const r3d_akaze_options* opt,
                           float* arrays, float* kcontrast, r3d_akaze_keypoint* cands, uint8_t* flags, uint32_t cand_cap,
                           uint32_t* cand_counts);

/* Diagnostics: one image through R3D_DETECTOR_AKAZE's kernels.  arrays / kcontrast as r3d_debug_akaze_levels;
 * masks: per level, in level order, three width x height uint8 masks of the kept points (1 = kept): after the
 * same-level pass, after the lower-level passes, after the upper-level passes. */
int r3d_debug_akaze_masks(r3d_ctx* ctx, const float* image, uint32_t width, uint32_t height, const r3d_akaze_options* opt,
                          float* arrays, float* kcontrast, uint8_t* masks);

/* Diagnostics: the subpixel refinement kernel alone on n points of one level (its Ldet, width x height, octave ratio):
 * out = the refined points; a rejected point (|d| > 1) is returned unchanged with class_id -1.  A singular 2x2
 * system solves to d = 0, as cv::solve leaves it. */
int r3d_debug_akaze_refine(r3d_ctx* ctx, const float* ldet, uint32_t width, uint32_t height, float ratio,
                           const r3d_akaze_keypoint* in, uint32_t n, r3d_akaze_keypoint* out);

/* ---- feature extraction (SURVEY.md 3: the feature stage, detector + descriptor + files) ------------------------- */
/* R3DFeaturesThread::extractFeaturesAndDescriptors for the "Fast-AKAZE" detector list (Regard3D's default,
 * src/Regard3DFeatures.cpp:133): per image detectAndExtract (:206-222) = the Fast-AKAZE branch (:590-614) +
 * extractLIOPFeatures (:719-861), then KeypointSet::saveToBinFile (src/threads/R3DFeaturesThread.cpp:200). */
typedef struct {
  r3d_akaze_options akaze;        /* threshold = R3DFParams::threshold_ */
  float kp_size_factor;           /* 8: getKpSizeFactor("Fast-AKAZE") and getKpSizeFactor("AKAZE"), :691-716 */
  const char* out_dir;            /* NULL: no files; else <out_dir>/<basenames[i]>.feat / .desc */
  const char* const* basenames;   /* n_images names without extension; required when out_dir is set */
} r3d_extract_options;
void r3d_extract_default_options(r3d_extract_options* out);
/* Each image is uploaded once; its keypoints (r3d_akaze_detect's, in upstream order) are described with LIOP
 * (r3d_liop_describe's kernel and bits) while it is still resident, and the descriptors of a batch are computed on a
 * second stream while the next batch builds its scale space.  With out_dir set, one host thread per device writes
 * <basename>.feat / .desc in OpenMVG's layout (r3d_save_features) while the device goes on.  The images are dealt to the
 * context's devices as r3d_akaze_detect deals them; the result does not depend on the number of devices.
 * R3D_ERR_INVALID before any work or file for everything r3d_akaze_detect rejects, a kp_size_factor that is not finite
 * and > 0, an empty out_dir, a missing or empty basename, or out == NULL without out_dir.  A file that cannot be
 * written: R3D_ERR_IO naming the path (files written before stay on disk).  cb (may be NULL) receives
 * 0.2 + 0.4 * done / n_images, message "", each time an image is finished (its files written when out_dir is set), as
 * src/threads/R3DFeaturesThread.cpp:211-228 does; never concurrently, never decreasing.  out (may be NULL when out_dir
 * is set): per image in image order, the keypoints (r3d_features_get) and their descriptors (r3d_features_descriptors);
 * r3d_features_count is the reference's numberOfKeypoints_ entry of the image -- the reference lists those in
 * thread-completion order, here they are in image order. */
int r3d_extract_features(r3d_ctx* ctx, const float* const* images, const uint32_t* widths, const uint32_t* heights,
                         uint32_t n_images, const r3d_extract_options* opt, r3d_progress_cb cb, void* user,
                         r3d_features** out);
/* r3d_extract_features with a choice of detector (R3D_DETECTOR_*; r3d_extract_features is R3D_DETECTOR_FAST_AKAZE):
 * the same arguments, rejections and outputs; an unknown detector is R3D_ERR_INVALID.  AKAZE keypoints are described
 * with their angle as cv::AKAZE returns it, as Regard3D's "AKAZE" list does. */
int r3d_extract_features_detector(r3d_ctx* ctx, int detector, const float* const* images, const uint32_t* widths,
                                  const uint32_t* heights, uint32_t n_images, const r3d_extract_options* opt,
                                  r3d_progress_cb cb, void* user, r3d_features** out);
/* count x 144 float32 in keypoint order; NULL for r3d_akaze_detect results and for images without keypoints */
const float* r3d_features_descriptors(const r3d_features* f, uint32_t image);
/* Host only: KeypointSet::saveToBinFile = openMVG saveFeatsToFile + saveDescsToBinFile.  feat_path: one line
 * "x y scale orientation\n" per keypoint (std::ostream <<, precision 6, classic locale); desc_path: a size_t count, then
 * n x dim float32.  xyso: n x 4 = x, y, scale (= size / 2), orientation (degrees).  R3D_ERR_IO naming the path. */
int r3d_save_features(const char* feat_path, const char* desc_path, const float* xyso, const float* desc, uint64_t n,
                      uint32_t dim);
/* the last r3d_extract_features: device stage times (CUDA events, summed over batches and devices), the host time of
 * the descriptor downloads and of the file writing (summed over the writer threads), the call's wall time */
typedef struct {
  double upload_ms;   /* images host -> device, workspace clears */
  double detect_ms;   /* r3d_akaze_timing's stages after the upload */
  double describe_ms; /* k_liop on the second stream */
  double d2h_ms;      /* descriptors device -> host */
  double write_ms;    /* .feat / .desc formatting and writing */
  double total_ms;
  uint32_t images, batches, keypoints, kernel_launches, devices;
} r3d_extract_timing;
int r3d_get_extract_timing(const r3d_ctx* ctx, r3d_extract_timing* out);

#ifdef __cplusplus
}
#endif
#endif /* R3DGPU_H */
