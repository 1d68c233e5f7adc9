"""ctypes binding of libr3dgpu.so (include/r3dgpu.h).

Fails loudly: importing works anywhere (the CPU-only tests check the exported symbols), but
`Context()` raises R3DError when no sm_90 device is present -- there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("R3D_LIB") or os.path.join(_HERE, "libr3dgpu.so")  # R3D_LIB: an A/B build of the same ABI

R3D_F32, R3D_U8 = 0, 1
MATCH_DEFAULT, MATCH_EXACT_SCAN, MATCH_NO_COORD_DEDUP, MATCH_MUTUAL_NN, MATCH_CASCADE_HASHING = 0, 1, 2, 4, 8
MATCHING_CASCADE_HASHING = 100  # r3d_cm_params.matching_algorithm extension
MODEL_F, MODEL_E, MODEL_H = 0, 1, 2

indmatch_dtype = np.dtype([("i", np.uint32), ("j", np.uint32)])

EXPORTS = [
    "r3d_create", "r3d_destroy", "r3d_last_error", "r3d_abi_version", "r3d_upload_regions",
    "r3d_clear_regions", "r3d_match_pairs", "r3d_search_neighbours", "r3d_matches_num_pairs",
    "r3d_matches_total", "r3d_matches_get_pair", "r3d_matches_from_csr", "r3d_free_matches",
    "r3d_save_matches_txt", "r3d_load_matches_txt", "r3d_filter_pairs", "r3d_ba_default_options",
    "r3d_bundle_adjust", "r3d_ba_residuals", "r3d_compute_matches", "r3d_get_match_timing",
    "r3d_get_filter_timing", "r3d_debug_candidate_keys", "r3d_debug_ba_jacobian",
    "r3d_comm_unique_id", "r3d_comm_init", "r3d_comm_destroy", "r3d_comm_world", "r3d_debug_post_process",
    "r3d_debug_post_process_many", "r3d_debug_post_process_ranked", "r3d_matches_export_csr", "r3d_debug_rng_selftest", "r3d_liop_describe", "r3d_debug_liop_process",
    "r3d_save_matches_bin", "r3d_load_matches_bin", "r3d_save_matches", "r3d_load_matches", "r3d_sfm_data_create",
    "r3d_sfm_data_free", "r3d_sfm_data_load", "r3d_sfm_data_save", "r3d_sfm_root_path", "r3d_sfm_set_root_path",
    "r3d_sfm_num_views", "r3d_sfm_num_intrinsics", "r3d_sfm_num_poses", "r3d_sfm_num_landmarks", "r3d_sfm_add_view",
    "r3d_sfm_get_view", "r3d_sfm_add_intrinsic", "r3d_sfm_get_intrinsic", "r3d_sfm_add_pose", "r3d_sfm_get_pose",
    "r3d_sfm_add_landmark", "r3d_sfm_get_landmark", "r3d_debug_ba_jacobian_model", "r3d_debug_ba_prior", "r3d_sfm_ba_default_options", "r3d_sfm_bundle_adjust",
    "r3d_tracks_build", "r3d_tracks_count", "r3d_tracks_get", "r3d_tracks_in_images", "r3d_tracks_free",
    "r3d_sfm_structure_from_tracks", "r3d_sfm_remove_outliers", "r3d_cascade_prepare", "r3d_debug_cascade_view",
    "r3d_relpose_default_options", "r3d_relative_poses", "r3d_get_relpose_timing",
    "r3d_resection_default_options", "r3d_resect_views", "r3d_sfm_resect_views", "r3d_get_resection_timing",
    "r3d_rotavg_default_options", "r3d_rotation_averaging", "r3d_rotavg_l1_default_options", "r3d_rotation_averaging_l1",
    "r3d_debug_rotavg_l1_step", "r3d_matches_keep_largest_biedge_component",
    "r3d_transavg_default_options", "r3d_translation_averaging", "r3d_transavg_l1_default_options",
    "r3d_translation_averaging_l1", "r3d_debug_transavg_l1_step", "r3d_debug_cholesky", "r3d_debug_chol_solve3",
    "r3d_debug_acransac_score", "r3d_debug_detmath", "r3d_debug_ba_step",
    "r3d_akaze_default_options", "r3d_akaze_levels", "r3d_akaze_detect", "r3d_features_num_images", "r3d_features_count",
    "r3d_features_get", "r3d_free_features", "r3d_get_akaze_timing", "r3d_debug_akaze_levels",
    "r3d_debug_akaze_refine", "r3d_debug_view_operands",
    "r3d_extract_default_options", "r3d_extract_features", "r3d_features_descriptors", "r3d_save_features",
    "r3d_get_extract_timing", "r3d_detect_keypoints", "r3d_extract_features_detector", "r3d_debug_akaze_masks",
    "r3d_sfm_colorize_plan", "r3d_sfm_write_colorized_ply", "r3d_undistort_images",
]

CHOL_DENSE, CHOL_ENVELOPE = 0, 1
# r3d_debug_ba_step: the Schur route (default plan, or every point through the CTA-per-point kernel)
SCHUR_PLAN, SCHUR_CTA = 0, 1
# r3d_ac_score: one model's scores from r3d_debug_acransac_score
ac_score_dtype = np.dtype([("lb", np.float64), ("nfa", np.float64), ("err", np.float64), ("cnt_hi", np.uint32),
                           ("cnt_lo", np.uint32), ("count", np.uint32), ("k", np.uint32)])
DETMATH_LOG10, DETMATH_CBRT, DETMATH_COS, DETMATH_ACOS = 0, 1, 2, 3


AKAZE_DIFF_PM_G2 = 1
# r3d_detect_keypoints / r3d_extract_features_detector: Regard3D's "Fast-AKAZE" and "AKAZE" detectors
DETECTOR_FAST_AKAZE, DETECTOR_AKAZE = 0, 1
# r3d_akaze_keypoint: angle in degrees after Regard3D's conversion; class_id = evolution level
akaze_keypoint_dtype = np.dtype([("x", np.float32), ("y", np.float32), ("size", np.float32), ("angle", np.float32),
                                 ("response", np.float32), ("octave", np.int32), ("class_id", np.int32)])
akaze_level_dtype = np.dtype([("octave", np.int32), ("sublevel", np.int32), ("width", np.int32), ("height", np.int32),
                              ("sigma_size", np.int32), ("border", np.int32), ("esigma", np.float32),
                              ("etime", np.float32), ("ratio", np.float32), ("n_tau", np.uint32)])
AKAZE_ARRAYS = ("Lt", "Lsmooth", "Lx", "Ly", "Ldet")


class AkazeOptions(C.Structure):
    _fields_ = [("threshold", C.c_float), ("octaves", C.c_int32), ("sublevels", C.c_int32), ("diffusivity", C.c_int32)]


class AkazeTiming(C.Structure):
    _fields_ = [("upload_ms", C.c_double), ("scale_space_ms", C.c_double), ("candidates_ms", C.c_double), ("same_level_ms", C.c_double),
                ("cross_level_ms", C.c_double), ("refine_orient_ms", C.c_double), ("total_ms", C.c_double),
                ("images", C.c_uint32), ("batches", C.c_uint32), ("keypoints", C.c_uint32),
                ("kernel_launches", C.c_uint32), ("devices", C.c_uint32)]


class ExtractOptions(C.Structure):
    _fields_ = [("akaze", AkazeOptions), ("kp_size_factor", C.c_float), ("out_dir", C.c_char_p),
                ("basenames", C.POINTER(C.c_char_p))]


class ExtractTiming(C.Structure):
    _fields_ = [("upload_ms", C.c_double), ("detect_ms", C.c_double), ("describe_ms", C.c_double), ("d2h_ms", C.c_double),
                ("write_ms", C.c_double), ("total_ms", C.c_double), ("images", C.c_uint32), ("batches", C.c_uint32),
                ("keypoints", C.c_uint32), ("kernel_launches", C.c_uint32), ("devices", C.c_uint32)]


def save_features(feat_path, desc_path, keypoints, descriptors):
    """Host only (no GPU): KeypointSet::saveToBinFile.  keypoints: akaze_keypoint_dtype, or (n, 4) float32 x, y, scale,
    orientation (scale = size / 2); descriptors (n, dim) float32."""
    if isinstance(keypoints, np.ndarray) and keypoints.dtype == akaze_keypoint_dtype:
        xyso = np.stack([keypoints["x"], keypoints["y"], keypoints["size"] / np.float32(2), keypoints["angle"]], 1)
    else:
        xyso = keypoints
    xyso = np.ascontiguousarray(xyso, np.float32).reshape(-1, 4)
    desc = np.ascontiguousarray(descriptors, np.float32)
    dim = desc.shape[1] if desc.ndim == 2 and desc.shape[1] else 144
    rc = lib().r3d_save_features(os.fsencode(feat_path), os.fsencode(desc_path), _p(xyso), _p(desc), C.c_uint64(len(xyso)),
                                 C.c_uint32(dim))
    if rc:
        raise R3DError(rc, lib().r3d_last_error(None).decode())


def akaze_options(threshold=0.001, octaves=4, sublevels=4, diffusivity=AKAZE_DIFF_PM_G2):
    o = AkazeOptions()
    lib().r3d_akaze_default_options(C.byref(o))
    o.threshold, o.octaves, o.sublevels, o.diffusivity = threshold, octaves, sublevels, diffusivity
    return o


def akaze_levels(width, height, **opts):
    """The detector's level table of a width x height image (akaze_level_dtype)."""
    out = np.zeros(64, akaze_level_dtype)
    n = lib().r3d_akaze_levels(C.c_uint32(width), C.c_uint32(height), C.byref(akaze_options(**opts)), _p(out), C.c_int(64))
    if n < 0:
        raise R3DError(n, "r3d_akaze_levels: bad arguments")
    return out[:n].copy()


class R3DError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libr3dgpu error %d: %s" % (code, msg))
        self.code = code


class MatchTiming(C.Structure):
    _fields_ = [("ms_prep", C.c_double), ("ms_candidates", C.c_double), ("ms_rerank", C.c_double),
                ("ms_fallback", C.c_double), ("ms_device_total", C.c_double), ("ms_host_post", C.c_double),
                ("kernel_launches", C.c_uint64), ("queries", C.c_uint64), ("fallback_queries", C.c_uint64),
                ("third_chunk_queries", C.c_uint64), ("fifth_chunk_queries", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("rejected_queries", C.c_uint64)]


class FilterTiming(C.Structure):
    _fields_ = [("ms_solve", C.c_double), ("ms_score", C.c_double), ("ms_device_total", C.c_double),
                ("ms_host", C.c_double), ("kernel_launches", C.c_uint64), ("hypotheses", C.c_uint64),
                ("rounds", C.c_uint64)]


class ViewInfo(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("focal", C.c_double), ("ppx", C.c_double),
                ("ppy", C.c_double)]


def make_views(widths, heights, Ks=None):
    """r3d_view_info array.  Ks: n x 3 (focal, ppx, ppy); default = R3DProject's approximation
    (src/R3DProject.cpp:1149-1159): focal = 1.1 * max(w, h), principal point at the image centre."""
    n = len(widths)
    views = (ViewInfo * n)()
    for k in range(n):
        w, h = int(widths[k]), int(heights[k])
        views[k].width, views[k].height = w, h
        if Ks is None:
            views[k].focal, views[k].ppx, views[k].ppy = 1.1 * max(w, h), w / 2.0, h / 2.0
        else:
            views[k].focal, views[k].ppx, views[k].ppy = float(Ks[k][0]), float(Ks[k][1]), float(Ks[k][2])
    return views


class BAProblem(C.Structure):
    _fields_ = [("n_cams", C.c_uint32), ("n_pts", C.c_uint32), ("n_intr", C.c_uint32), ("n_obs", C.c_uint64),
                ("poses", C.c_void_p), ("intrinsics", C.c_void_p), ("points", C.c_void_p),
                ("obs_cam", C.c_void_p), ("obs_pt", C.c_void_p), ("cam_intr", C.c_void_p),
                ("obs_xy", C.c_void_p),
                ("intr_model", C.c_void_p), ("intrinsics_ext", C.c_void_p), ("n_priors", C.c_uint32),
                ("prior_cam", C.c_void_p), ("prior_center", C.c_void_p), ("prior_weight", C.c_void_p)]


class BAOptions(C.Structure):
    _fields_ = [("max_iterations", C.c_uint32), ("huber_a", C.c_double), ("refine_intrinsics", C.c_int),
                ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("parameter_tolerance", C.c_double), ("initial_radius", C.c_double), ("prior_huber_a", C.c_double)]


class BASummary(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("successful_steps", C.c_uint32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("termination", C.c_int), ("seconds_total", C.c_double),
                ("seconds_linear", C.c_double), ("seconds_setup", C.c_double)]


class BAStepOut(C.Structure):
    _fields_ = [("g", C.c_void_p), ("diag", C.c_void_p), ("scale", C.c_void_p), ("S", C.c_void_p), ("rhs", C.c_void_p),
                ("Vinv", C.c_void_p), ("delta", C.c_void_p), ("nB", C.c_uint32), ("n_batches", C.c_uint32),
                ("n_long", C.c_uint32), ("not_pd", C.c_int), ("gmax", C.c_double), ("model_cost_change", C.c_double),
                ("dx_norm2", C.c_double), ("x_norm2", C.c_double)]


class RelposeOptions(C.Structure):
    _fields_ = [("precision_px", C.c_double), ("max_iter", C.c_uint32), ("refine", C.c_int), ("ba", BAOptions)]


RELPOSE_OK, RELPOSE_TOO_FEW, RELPOSE_NO_INTRINSIC, RELPOSE_NO_MODEL, RELPOSE_CHEIRALITY = 0, 1, 2, 3, 4
# r3d_relative_pose
relpose_dtype = np.dtype([
    ("I", np.uint32), ("J", np.uint32), ("status", np.int32), ("n_inliers", np.uint32),
    ("found_residual_precision", np.float64), ("E", np.float64, (3, 3)), ("rotation", np.float64, (3, 3)),
    ("translation", np.float64, 3), ("ba_iterations", np.uint32), ("ba_successful_steps", np.uint32),
    ("ba_termination", np.int32), ("ba_initial_cost", np.float64), ("ba_final_cost", np.float64)], align=True)


class RelposeTiming(C.Structure):
    _fields_ = [("ms_ransac", C.c_double), ("ms_cheirality", C.c_double), ("ms_refine", C.c_double),
                ("ms_device_total", C.c_double), ("ms_host", C.c_double), ("kernel_launches", C.c_uint64),
                ("ba_iterations", C.c_uint64)]


ROTAVG_L2, ROTAVG_L1 = 0, 1
ROTAVG_MAX_VIEWS = 4096


class RotavgOptions(C.Structure):
    _fields_ = [("method", C.c_int), ("max_angular_error_deg", C.c_double), ("refine", C.c_int), ("lm", BAOptions)]


class RotavgSummary(C.Structure):
    _fields_ = [("success", C.c_int), ("n_edges", C.c_uint64), ("n_triplets", C.c_uint64), ("n_valid_triplets", C.c_uint64),
                ("n_kept_edges", C.c_uint64), ("n_kept_views", C.c_uint32), ("init_iterations", C.c_uint32),
                ("lm_iterations", C.c_uint32), ("lm_successful_steps", C.c_uint32), ("lm_termination", C.c_int),
                ("lm_initial_cost", C.c_double), ("lm_final_cost", C.c_double), ("ms_triplets", C.c_double),
                ("ms_init", C.c_double), ("ms_refine", C.c_double), ("ms_device_total", C.c_double), ("ms_host", C.c_double)]


class RotavgL1Options(C.Structure):
    _fields_ = [("max_angular_error_deg", C.c_double), ("irls_sigma_deg", C.c_double), ("l1_max_iterations", C.c_int),
                ("irls_max_iterations", C.c_int), ("tolerance", C.c_double)]


class RotavgL1Summary(C.Structure):
    _fields_ = [("success", C.c_int), ("n_edges", C.c_uint64), ("n_triplets", C.c_uint64), ("n_valid_triplets", C.c_uint64),
                ("n_kept_edges", C.c_uint64), ("n_kept_views", C.c_uint32), ("l1_iterations", C.c_uint32),
                ("pd_iterations", C.c_uint32), ("pd_backtracks", C.c_uint32), ("irls_iterations", C.c_uint32),
                ("termination", C.c_int), ("initial_l1_cost", C.c_double), ("final_l1_cost", C.c_double),
                ("ms_triplets", C.c_double), ("ms_init", C.c_double), ("ms_l1", C.c_double), ("ms_irls", C.c_double),
                ("ms_device_total", C.c_double), ("ms_host", C.c_double)]


class RotavgL1StepOut(C.Structure):
    _fields_ = [("n_kept_views", C.c_uint32), ("n_kept_edges", C.c_uint32), ("view_ids", C.c_void_p), ("ab", C.c_void_p),
                ("Rk", C.c_void_p), ("rotations0", C.c_void_p), ("b", C.c_void_p), ("cost", C.c_void_p), ("bmax", C.c_double),
                ("b_zero", C.c_int), ("state0", C.c_void_p), ("sdg0", C.c_double), ("tau0", C.c_double),
                ("resnorm0", C.c_double), ("sigx", C.c_void_p), ("rrow", C.c_void_p), ("w2", C.c_void_p),
                ("laplacians", C.c_void_p), ("not_pd", C.c_int), ("dx", C.c_void_p), ("Adx", C.c_void_p), ("du", C.c_void_p),
                ("dl1", C.c_void_p), ("dl2", C.c_void_p), ("Atdv", C.c_void_p), ("rmin", C.c_void_p), ("step_max", C.c_double),
                ("n_trials", C.c_uint32), ("trial_step", C.c_double * 33), ("trial_resnorm", C.c_double * 33),
                ("accepted", C.c_int), ("state", C.c_void_p), ("sdg", C.c_double), ("tau", C.c_double),
                ("resnorm", C.c_double), ("w", C.c_void_p), ("wb", C.c_void_p), ("rotations", C.c_void_p),
                ("xmax", C.c_double), ("sys_not_pd", C.c_void_p)]


TRANSAVG_L1, TRANSAVG_L2_CHORDAL, TRANSAVG_SOFTL1 = 1, 2, 3


class TransavgOptions(C.Structure):
    _fields_ = [("method", C.c_int), ("softl1_loss", C.c_double), ("lm", BAOptions)]


class TransavgSummary(C.Structure):
    _fields_ = [("success", C.c_int), ("n_edges", C.c_uint64), ("n_kept_edges", C.c_uint64), ("n_kept_views", C.c_uint32),
                ("lm_iterations", C.c_uint32), ("lm_successful_steps", C.c_uint32), ("lm_termination", C.c_int),
                ("lm_initial_cost", C.c_double), ("lm_final_cost", C.c_double), ("ms_solve", C.c_double),
                ("ms_device_total", C.c_double), ("ms_host", C.c_double)]


class TransavgL1Options(C.Structure):
    _fields_ = [("max_iterations", C.c_int), ("tolerance", C.c_double)]


class TransavgL1Summary(C.Structure):
    _fields_ = [("success", C.c_int), ("n_edges", C.c_uint64), ("n_kept_edges", C.c_uint64), ("n_kept_views", C.c_uint32),
                ("iterations", C.c_uint32), ("regularized_factorizations", C.c_uint32), ("termination", C.c_int),
                ("gamma", C.c_double), ("dual_objective", C.c_double), ("max_primal_violation", C.c_double),
                ("max_dual_violation", C.c_double), ("ms_solve", C.c_double), ("ms_device_total", C.c_double),
                ("ms_host", C.c_double)]


class TransavgL1StepOut(C.Structure):
    _fields_ = [("n_kept_views", C.c_uint32), ("n_kept_edges", C.c_uint32), ("n", C.c_uint32), ("view_ids", C.c_void_p),
                ("edge_record", C.c_void_p), ("edge_ij", C.c_void_p), ("Rij", C.c_void_p), ("u", C.c_void_p),
                ("state0", C.c_void_p), ("norms", C.c_double * 5), ("A", C.c_void_p), ("sc", C.c_void_p),
                ("not_pd", C.c_int * 6), ("retries", C.c_uint32), ("pred_dy", C.c_void_p), ("pred_dlam", C.c_void_p),
                ("pred_ds", C.c_void_p), ("pred_dz", C.c_void_p), ("pred_alpha_p", C.c_double), ("pred_alpha_d", C.c_double),
                ("pred_complementarity", C.c_double), ("sigma", C.c_double), ("corr_rhs", C.c_void_p),
                ("corr_dy", C.c_void_p), ("corr_dlam", C.c_void_p), ("corr_ds", C.c_void_p), ("corr_dz", C.c_void_p),
                ("alpha_p", C.c_double), ("alpha_d", C.c_double), ("state", C.c_void_p), ("converged", C.c_int),
                ("failed", C.c_int)]


def relative_pose_records(I, J, R, status=None):
    """r3d_relative_pose records (relpose_dtype) from view ids and rotations (X_J = R X_I + t), e.g. for
    Context.rotation_averaging on relative motions that did not come from relative_poses."""
    I = np.asarray(I, np.uint32).ravel()
    rel = np.zeros(len(I), relpose_dtype)
    rel["I"] = I
    rel["J"] = np.asarray(J, np.uint32).ravel()
    rel["rotation"] = np.asarray(R, np.float64).reshape(-1, 3, 3)
    rel["status"] = RELPOSE_OK if status is None else np.asarray(status, np.int32)
    rel["ba_termination"] = -1
    return rel


class CMParams(C.Structure):
    _fields_ = [("dist_ratio", C.c_float), ("compute_fundamental", C.c_int), ("compute_essential", C.c_int),
                ("compute_homography", C.c_int), ("matching_algorithm", C.c_int), ("descriptor_dim", C.c_uint32),
                ("svg_output", C.c_int)]


class CMPaths(C.Structure):
    _fields_ = [("matches_dir", C.c_char_p), ("image_basenames", C.POINTER(C.c_char_p)),
                ("views", C.POINTER(ViewInfo)), ("n_views", C.c_uint32), ("matches_f_filename", C.c_char_p),
                ("matches_h_filename", C.c_char_p), ("matches_e_filename", C.c_char_p)]


class CMStats(C.Structure):
    _fields_ = [("n_views", C.c_uint32), ("number_of_keypoints", C.POINTER(C.c_uint32)),
                ("putative_pairs", C.c_uint64), ("putative_matches", C.c_uint64), ("f_pairs", C.c_uint64),
                ("f_matches", C.c_uint64), ("h_pairs", C.c_uint64), ("h_matches", C.c_uint64), ("e_pairs", C.c_uint64),
                ("e_matches", C.c_uint64), ("seconds_load", C.c_double), ("seconds_match", C.c_double),
                ("seconds_filter", C.c_double)]


PROGRESS_CB = C.CFUNCTYPE(None, C.c_float, C.c_char_p, C.c_void_p)

_lib = None


def lib():
    """Load libr3dgpu.so (raises if it has not been built: `python -m regard3d_b200.build`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("libr3dgpu.so is not built; run `python -m regard3d_b200.build` "
                              "(there is no fallback implementation)")
        L = C.CDLL(LIB_PATH)
        L.r3d_last_error.restype = C.c_char_p
        L.r3d_last_error.argtypes = [C.c_void_p]
        L.r3d_features_count.restype = C.c_uint32
        L.r3d_features_count.argtypes = [C.c_void_p, C.c_uint32]
        L.r3d_features_get.restype = C.c_void_p
        L.r3d_features_get.argtypes = [C.c_void_p, C.c_uint32]
        L.r3d_free_features.argtypes = [C.c_void_p]
        L.r3d_features_descriptors.restype = C.c_void_p
        L.r3d_features_descriptors.argtypes = [C.c_void_p, C.c_uint32]
        L.r3d_matches_num_pairs.restype = C.c_uint64
        L.r3d_matches_num_pairs.argtypes = [C.c_void_p]
        L.r3d_matches_total.restype = C.c_uint64
        L.r3d_matches_total.argtypes = [C.c_void_p]
        L.r3d_free_matches.argtypes = [C.c_void_p]
        L.r3d_destroy.argtypes = [C.c_void_p]
        L.r3d_sfm_data_free.argtypes = [C.c_void_p]
        L.r3d_sfm_root_path.restype = C.c_char_p
        L.r3d_sfm_root_path.argtypes = [C.c_void_p]
        for fn in (L.r3d_sfm_num_views, L.r3d_sfm_num_intrinsics, L.r3d_sfm_num_poses):
            fn.restype = C.c_uint32
            fn.argtypes = [C.c_void_p]
        L.r3d_sfm_num_landmarks.restype = C.c_uint32
        L.r3d_sfm_num_landmarks.argtypes = [C.c_void_p, C.c_int]
        L.r3d_sfm_data_save.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32]
        L.r3d_sfm_set_root_path.argtypes = [C.c_void_p, C.c_char_p]
        L.r3d_sfm_add_view.argtypes = [C.c_void_p, C.c_void_p]
        L.r3d_sfm_get_view.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.r3d_sfm_add_intrinsic.argtypes = [C.c_void_p, C.c_void_p]
        L.r3d_sfm_get_intrinsic.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.r3d_sfm_add_pose.argtypes = [C.c_void_p, C.c_void_p]
        L.r3d_sfm_get_pose.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.r3d_sfm_add_landmark.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32]
        L.r3d_sfm_get_landmark.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        L.r3d_tracks_count.restype = C.c_uint64
        L.r3d_tracks_count.argtypes = [C.c_void_p]
        L.r3d_tracks_free.argtypes = [C.c_void_p]
        L.r3d_tracks_build.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.r3d_tracks_get.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.r3d_tracks_in_images.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        L.r3d_sfm_structure_from_tracks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.r3d_sfm_remove_outliers.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_uint32, C.c_double, C.c_void_p, C.c_void_p]
        L.r3d_sfm_bundle_adjust.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.r3d_sfm_colorize_plan.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.r3d_sfm_write_colorized_ply.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p]
        L.r3d_undistort_images.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p]
        L.r3d_save_matches.argtypes = [C.c_void_p, C.c_char_p]
        L.r3d_save_matches_bin.argtypes = [C.c_void_p, C.c_char_p]
        L.r3d_comm_world.argtypes = [C.c_void_p]
        L.r3d_resect_views.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]
        L.r3d_sfm_resect_views.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.r3d_debug_post_process.restype = C.c_int64
        L.r3d_debug_post_process_ranked.restype = C.c_int64
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Matches:
    """PairWiseMatches handle (openMVG::matching::PairWiseMatches)."""

    def __init__(self, handle):
        self.handle = C.c_void_p(handle) if not isinstance(handle, C.c_void_p) else handle

    def __del__(self):
        try:
            if self.handle:
                lib().r3d_free_matches(self.handle)
                self.handle = None
        except Exception:
            pass

    @property
    def num_pairs(self):
        return int(lib().r3d_matches_num_pairs(self.handle))

    @property
    def total(self):
        return int(lib().r3d_matches_total(self.handle))

    def pair(self, k):
        I, J = C.c_uint32(), C.c_uint32()
        ptr = C.c_void_p()
        cnt = C.c_uint64()
        rc = lib().r3d_matches_get_pair(self.handle, C.c_uint64(k), C.byref(I), C.byref(J), C.byref(ptr), C.byref(cnt))
        if rc:
            raise R3DError(rc, "r3d_matches_get_pair")
        n = cnt.value
        if n == 0:
            return I.value, J.value, np.zeros(0, indmatch_dtype)
        buf = (C.c_uint8 * (8 * n)).from_address(ptr.value)
        return I.value, J.value, np.frombuffer(buf, dtype=indmatch_dtype).copy()

    def to_dict(self):
        out = {}
        for k in range(self.num_pairs):
            I, J, m = self.pair(k)
            out[(I, J)] = m
        return out

    def to_csr(self, pairs):
        """CSR over the caller's pair list (empty range for pairs absent from the map)."""
        d = self.to_dict()
        pairs = np.asarray(pairs, np.uint32).reshape(-1, 2)
        ofs = np.zeros(len(pairs) + 1, np.uint64)
        chunks = []
        for k, (I, J) in enumerate(pairs):
            m = d.get((int(I), int(J)))
            n = 0 if m is None else len(m)
            ofs[k + 1] = ofs[k] + n
            if n:
                chunks.append(m)
        allm = np.concatenate(chunks) if chunks else np.zeros(0, indmatch_dtype)
        return ofs, allm

    def export_csr(self, pairs_out=None, ofs_out=None, matches_out=None):
        """(pairs[P,2] u32, ofs[P+1] u64, matches[total]) in map order -- one memcpy per pair inside the library.
        Caller buffers (e.g. pinned torch tensors viewed as numpy) may be passed to avoid allocations."""
        P, T = self.num_pairs, self.total
        if pairs_out is None:
            pairs_out = np.empty((P, 2), np.uint32)
        if ofs_out is None:
            ofs_out = np.empty(P + 1, np.uint64)
        if matches_out is None:
            matches_out = np.empty(T, indmatch_dtype)
        assert pairs_out.size >= 2 * P and ofs_out.size >= P + 1 and matches_out.size >= T
        rc = lib().r3d_matches_export_csr(self.handle, _p(pairs_out), _p(ofs_out), _p(matches_out))
        if rc:
            raise R3DError(rc, "r3d_matches_export_csr")
        return pairs_out, ofs_out, matches_out

    def save(self, path):
        """matching::Save: '.txt' or '.bin' (cereal portable binary) by extension."""
        rc = lib().r3d_save_matches(self.handle, path.encode())
        if rc:
            raise R3DError(rc, "r3d_save_matches(%s)" % path)

    @staticmethod
    def load(path):
        h = C.c_void_p()
        rc = lib().r3d_load_matches(path.encode(), C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_load_matches(%s)" % path)
        return Matches(h)

    def save_txt(self, path):
        rc = lib().r3d_save_matches_txt(self.handle, path.encode())
        if rc:
            raise R3DError(rc, "r3d_save_matches_txt(%s)" % path)

    @staticmethod
    def load_txt(path):
        h = C.c_void_p()
        rc = lib().r3d_load_matches_txt(path.encode(), C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_load_matches_txt(%s)" % path)
        return Matches(h)

    def keep_largest_biedge_component(self):
        """graph::CleanGraph_KeepLargestBiEdge_Nodes + KeepOnlyReferencedElement: the pairs inside the largest
        2-edge-connected component of the pair graph (host only)."""
        h = C.c_void_p()
        rc = lib().r3d_matches_keep_largest_biedge_component(self.handle, C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_matches_keep_largest_biedge_component")
        return Matches(h)

    @staticmethod
    def from_csr(pairs, ofs, m):
        pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        ofs = np.ascontiguousarray(ofs, np.uint64)
        m = np.ascontiguousarray(m, indmatch_dtype)
        h = C.c_void_p()
        rc = lib().r3d_matches_from_csr(_p(pairs), C.c_uint64(len(pairs)), _p(ofs), _p(m), C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_matches_from_csr")
        return Matches(h)


class SfmView(C.Structure):
    _fields_ = [("id_view", C.c_uint32), ("id_intrinsic", C.c_uint32), ("id_pose", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("local_path", C.c_char_p), ("filename", C.c_char_p), ("has_prior", C.c_int),
                ("center_weight", C.c_double * 3), ("pose_center", C.c_double * 3)]


class SfmIntrinsic(C.Structure):
    _fields_ = [("id", C.c_uint32), ("model", C.c_int), ("width", C.c_uint32), ("height", C.c_uint32),
                ("focal", C.c_double), ("ppx", C.c_double), ("ppy", C.c_double), ("disto", C.c_double * 5)]


class SfmPose(C.Structure):
    _fields_ = [("id", C.c_uint32), ("rotation", C.c_double * 9), ("center", C.c_double * 3)]


class SfmObservation(C.Structure):
    _fields_ = [("id_view", C.c_uint32), ("id_feat", C.c_uint32), ("x", C.c_double * 2)]


SFM_VIEWS, SFM_EXTRINSICS, SFM_INTRINSICS, SFM_STRUCTURE, SFM_CONTROL_POINTS, SFM_ALL = 1, 2, 4, 8, 16, 31
CAM_PINHOLE, CAM_RADIAL1, CAM_RADIAL3, CAM_BROWN, CAM_FISHEYE = 1, 2, 3, 4, 5


class UndistortTiming(C.Structure):
    _fields_ = [("upload_ms", C.c_double), ("kernel_ms", C.c_double), ("download_ms", C.c_double), ("stage_ms", C.c_double),
                ("total_ms", C.c_double), ("images", C.c_uint32), ("copied", C.c_uint32), ("kernel_launches", C.c_uint32),
                ("devices", C.c_uint32)]


class ResectionOptions(C.Structure):
    _fields_ = [("precision_px", C.c_double), ("max_iter", C.c_uint32), ("refine", C.c_int), ("ba", BAOptions)]


class ResectionView(C.Structure):
    _fields_ = [("view_id", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32), ("intrinsic", SfmIntrinsic),
                ("first", C.c_uint64), ("count", C.c_uint64)]


class ResectionTiming(C.Structure):
    _fields_ = [("ms_ransac", C.c_double), ("ms_refine", C.c_double), ("ms_device_total", C.c_double), ("ms_host", C.c_double),
                ("kernel_launches", C.c_uint64), ("lm_iterations", C.c_uint64)]


RESECT_OK, RESECT_TOO_FEW, RESECT_NO_INTRINSIC, RESECT_NO_MODEL = 0, 1, 2, 3
resection_dtype = np.dtype([
    ("view_id", np.uint32), ("status", np.int32), ("n_inliers", np.uint32), ("found_residual_precision", np.float64),
    ("rotation", np.float64, (3, 3)), ("center", np.float64, 3), ("translation", np.float64, 3),
    ("rotation_ransac", np.float64, (3, 3)), ("translation_ransac", np.float64, 3), ("lm_iterations", np.uint32),
    ("lm_successful_steps", np.uint32), ("lm_termination", np.int32), ("lm_initial_cost", np.float64),
    ("lm_final_cost", np.float64)], align=True)


def resection_views(counts, widths, heights, models, focals, ppxs, ppys, distos=None, view_ids=None):
    """r3d_resection_view array for views whose correspondences lie one after the other in X / x."""
    n = len(counts)
    arr = (ResectionView * n)()
    first = 0
    for v in range(n):
        a = arr[v]
        a.view_id = int(view_ids[v]) if view_ids is not None else v
        a.width, a.height = int(widths[v]), int(heights[v])
        a.intrinsic.id = v
        a.intrinsic.model = int(models[v])
        a.intrinsic.width, a.intrinsic.height = int(widths[v]), int(heights[v])
        a.intrinsic.focal, a.intrinsic.ppx, a.intrinsic.ppy = float(focals[v]), float(ppxs[v]), float(ppys[v])
        if distos is not None:
            for i, d in enumerate(distos[v]):
                a.intrinsic.disto[i] = float(d)
        a.first, a.count = first, int(counts[v])
        first += int(counts[v])
    return arr


class SfmData:
    """openMVG::sfm::SfM_Data handle (sfm_data.bin: cereal portable binary, no OpenMVG needed)."""

    def __init__(self, handle=None):
        if handle is None:
            handle = C.c_void_p()
            rc = lib().r3d_sfm_data_create(C.byref(handle))
            if rc:
                raise R3DError(rc, "r3d_sfm_data_create")
        self.h = handle

    def __del__(self):
        try:
            if self.h:
                lib().r3d_sfm_data_free(self.h)
                self.h = None
        except Exception:
            pass

    @staticmethod
    def load(path):
        h = C.c_void_p()
        rc = lib().r3d_sfm_data_load(path.encode(), C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_sfm_data_load(%s)" % path)
        return SfmData(h)

    def save(self, path, parts=SFM_ALL):
        rc = lib().r3d_sfm_data_save(self.h, path.encode(), C.c_uint32(parts))
        if rc:
            raise R3DError(rc, "r3d_sfm_data_save(%s)" % path)

    @property
    def root_path(self):
        return lib().r3d_sfm_root_path(self.h).decode()

    @root_path.setter
    def root_path(self, p):
        lib().r3d_sfm_set_root_path(self.h, p.encode())

    def add_view(self, id_view, filename, width, height, id_intrinsic=None, id_pose=None, local_path="", prior_center=None,
                 prior_weight=(1.0, 1.0, 1.0)):
        v = SfmView(id_view, id_view if id_intrinsic is None else id_intrinsic, id_view if id_pose is None else id_pose,
                    width, height, local_path.encode(), filename.encode(), 0 if prior_center is None else 1,
                    (C.c_double * 3)(*prior_weight), (C.c_double * 3)(*(prior_center or (0.0, 0.0, 0.0))))
        rc = lib().r3d_sfm_add_view(self.h, C.byref(v))
        if rc:
            raise R3DError(rc, "r3d_sfm_add_view")

    def add_intrinsic(self, id, model, width, height, focal, ppx, ppy, disto=()):
        d = list(disto) + [0.0] * (5 - len(disto))
        s = SfmIntrinsic(id, model, width, height, focal, ppx, ppy, (C.c_double * 5)(*d))
        rc = lib().r3d_sfm_add_intrinsic(self.h, C.byref(s))
        if rc:
            raise R3DError(rc, "r3d_sfm_add_intrinsic")

    def add_pose(self, id, R, center):
        s = SfmPose(id, (C.c_double * 9)(*np.asarray(R, float).reshape(9)), (C.c_double * 3)(*np.asarray(center, float)))
        rc = lib().r3d_sfm_add_pose(self.h, C.byref(s))
        if rc:
            raise R3DError(rc, "r3d_sfm_add_pose")

    def add_landmark(self, id, X, obs, control_point=False):
        """obs: list of (id_view, id_feat, x, y)."""
        arr = (SfmObservation * max(len(obs), 1))()
        for k, (v, f, x, y) in enumerate(obs):
            arr[k] = SfmObservation(v, f, (C.c_double * 2)(x, y))
        rc = lib().r3d_sfm_add_landmark(self.h, C.c_int(int(control_point)), C.c_uint32(id), (C.c_double * 3)(*X), arr,
                                        C.c_uint32(len(obs)))
        if rc:
            raise R3DError(rc, "r3d_sfm_add_landmark")

    def views(self):
        out = []
        for k in range(lib().r3d_sfm_num_views(self.h)):
            v = SfmView()
            lib().r3d_sfm_get_view(self.h, C.c_uint32(k), C.byref(v))
            out.append(dict(id_view=v.id_view, id_intrinsic=v.id_intrinsic, id_pose=v.id_pose, width=v.width, height=v.height,
                            local_path=v.local_path.decode(), filename=v.filename.decode(), has_prior=bool(v.has_prior),
                            center_weight=list(v.center_weight), pose_center=list(v.pose_center)))
        return out

    def intrinsics(self):
        out = []
        for k in range(lib().r3d_sfm_num_intrinsics(self.h)):
            s = SfmIntrinsic()
            lib().r3d_sfm_get_intrinsic(self.h, C.c_uint32(k), C.byref(s))
            out.append(dict(id=s.id, model=s.model, width=s.width, height=s.height, focal=s.focal, ppx=s.ppx, ppy=s.ppy,
                            disto=list(s.disto)))
        return out

    def poses(self):
        out = []
        for k in range(lib().r3d_sfm_num_poses(self.h)):
            s = SfmPose()
            lib().r3d_sfm_get_pose(self.h, C.c_uint32(k), C.byref(s))
            out.append(dict(id=s.id, R=np.array(list(s.rotation)).reshape(3, 3), center=np.array(list(s.center))))
        return out

    def landmarks(self, control_points=False):
        out = []
        cp = C.c_int(int(control_points))
        for k in range(lib().r3d_sfm_num_landmarks(self.h, cp)):
            n = C.c_uint32()
            lid = C.c_uint32()
            X = (C.c_double * 3)()
            lib().r3d_sfm_get_landmark(self.h, cp, C.c_uint32(k), C.byref(lid), X, None, C.c_uint32(0), C.byref(n))
            arr = (SfmObservation * max(n.value, 1))()
            lib().r3d_sfm_get_landmark(self.h, cp, C.c_uint32(k), None, None, arr, n, None)
            out.append(dict(id=lid.value, X=list(X), obs=[(arr[q].id_view, arr[q].id_feat, arr[q].x[0], arr[q].x[1])
                                                          for q in range(n.value)]))
        return out

    def colorize(self, ctx, read_rgb):
        """OpenMVGHelper::ColorizeTracks: the colour of every landmark, (num_landmarks, 3) uint8 in landmark id order.
        The plan comes from the device (Context.colorize_plan); read_rgb(view_id) -> H x W x 3 uint8 is called once per
        round, in the order upstream reads the images, and only the planned pixels are gathered from each."""
        round_view, lm_round, lm_pixel = ctx.colorize_plan(self)
        sizes = {v["id_view"]: (v["height"], v["width"]) for v in self.views()}
        colors = np.zeros((len(lm_round), 3), np.uint8)
        for r, v in enumerate(round_view.tolist()):
            img = np.asarray(read_rgb(v))
            if img.dtype != np.uint8 or img.shape != sizes[v] + (3,):
                raise ValueError("read_rgb(%d): expected a %d x %d x 3 uint8 image, got %s %s"
                                 % ((v,) + sizes[v] + (img.dtype, img.shape)))
            sel = np.nonzero(lm_round == r)[0]
            colors[sel] = img[lm_pixel[sel, 1], lm_pixel[sel, 0]]
        return colors

    def write_colorized_ply(self, path, colors=None):
        """FinalColorized.ply: landmarks with colors ((num_landmarks, 3) uint8, None = white), then the pose centres."""
        col = None
        if colors is not None:
            col = np.ascontiguousarray(colors, np.uint8)
            if col.shape != (lib().r3d_sfm_num_landmarks(self.h, 0), 3):
                raise ValueError("colors: expected (num_landmarks, 3), got %s" % (col.shape,))
        rc = lib().r3d_sfm_write_colorized_ply(self.h, None if col is None else _p(col), path.encode())
        if rc:
            raise R3DError(rc, lib().r3d_last_error(None).decode())


class Tracks:
    """openMVG::tracks::STLMAPTracks handle (TracksBuilder Build + Filter + ExportToSTL)."""

    def __init__(self, handle):
        self.h = handle

    def __del__(self):
        try:
            if self.h:
                lib().r3d_tracks_free(self.h)
                self.h = None
        except Exception:
            pass

    @staticmethod
    def build(matches, min_length=2):
        h = C.c_void_p()
        rc = lib().r3d_tracks_build(matches.handle, C.c_uint32(min_length), C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_tracks_build")
        return Tracks(h)

    def __len__(self):
        return int(lib().r3d_tracks_count(self.h))

    def get(self, k):
        tid, n = C.c_uint32(), C.c_uint32()
        pv, pf = C.c_void_p(), C.c_void_p()
        rc = lib().r3d_tracks_get(self.h, C.c_uint64(k), C.byref(tid), C.byref(pv), C.byref(pf), C.byref(n))
        if rc:
            raise R3DError(rc, "r3d_tracks_get")
        v = np.frombuffer((C.c_uint32 * n.value).from_address(pv.value), np.uint32).copy() if n.value else np.zeros(0, np.uint32)
        f = np.frombuffer((C.c_uint32 * n.value).from_address(pf.value), np.uint32).copy() if n.value else np.zeros(0, np.uint32)
        return tid.value, v, f

    def to_dict(self):
        """{track id: {view: feature}} like STLMAPTracks."""
        out = {}
        for k in range(len(self)):
            tid, v, f = self.get(k)
            out[tid] = dict(zip(v.tolist(), f.tolist()))
        return out

    def in_images(self, view_ids):
        ids = np.ascontiguousarray(view_ids, np.uint32)
        h = C.c_void_p()
        rc = lib().r3d_tracks_in_images(self.h, _p(ids), C.c_uint32(len(ids)), C.byref(h))
        if rc:
            raise R3DError(rc, "r3d_tracks_in_images")
        return Tracks(h)


def debug_ba_jacobian_model(model, intr, ext, pose, X, obs):
    """Host evaluation of the analytic model of any of the five camera types (no GPU needed)."""
    intr, pose, X, obs = [np.ascontiguousarray(a, np.float64) for a in (intr, pose, X, obs)]
    ext = None if ext is None else np.ascontiguousarray(ext, np.float64)
    r = np.zeros(2)
    J = np.zeros((2, 15))
    rc = lib().r3d_debug_ba_jacobian_model(C.c_int(model), _p(intr), None if ext is None else _p(ext), _p(pose), _p(X), _p(obs),
                                           _p(r), _p(J))
    if rc:
        raise R3DError(rc, "r3d_debug_ba_jacobian_model")
    return r, J


def debug_detmath(fn, x, on_device):
    """r3d_debug_detmath: detmath.cuh's log10 / cbrt / cos / acos (DETMATH_*) of every entry of x, on the current CUDA
    device or in the library's host code."""
    x = np.ascontiguousarray(x, np.float64).ravel()
    y = np.empty_like(x)
    rc = lib().r3d_debug_detmath(C.c_int(fn), C.c_int(int(on_device)), _p(x), C.c_uint64(len(x)), _p(y))
    if rc:
        raise R3DError(rc, lib().r3d_last_error(None).decode())
    return y


def debug_ba_prior(pose, center, weight):
    pose, center, weight = [np.ascontiguousarray(a, np.float64) for a in (pose, center, weight)]
    r = np.zeros(3)
    J = np.zeros((3, 6))
    lib().r3d_debug_ba_prior(_p(pose), _p(center), _p(weight), _p(r), _p(J))
    return r, J


def debug_ba_jacobian(intr, pose, X, obs):
    """Host evaluation of the analytic BA model (no GPU needed)."""
    intr, pose, X, obs = [np.ascontiguousarray(a, np.float64) for a in (intr, pose, X, obs)]
    r = np.zeros(2)
    J = np.zeros((2, 15))
    lib().r3d_debug_ba_jacobian(_p(intr), _p(pose), _p(X), _p(obs), _p(r), _p(J))
    return r, J


class Context:
    """r3d_ctx: one per process / GPU in bench.py; device_ids selects the CUDA devices."""

    def __init__(self, device_ids=(0,)):
        self._h = C.c_void_p()
        ids = (C.c_int * len(device_ids))(*device_ids)
        rc = lib().r3d_create(ids, len(device_ids), C.byref(self._h))
        if rc:
            raise R3DError(rc, lib().r3d_last_error(None).decode())

    def close(self):
        if self._h:
            lib().r3d_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            raise R3DError(rc, lib().r3d_last_error(self._h).decode())

    def upload_regions(self, view_id, desc, xy=None):
        desc = np.ascontiguousarray(desc)
        if desc.dtype == np.float32:
            dt = R3D_F32
        elif desc.dtype == np.uint8:
            dt = R3D_U8
        else:
            raise TypeError("descriptors must be float32 or uint8")
        n, dim = (desc.shape[0], desc.shape[1]) if desc.ndim == 2 else (0, 0)
        xyp = None
        if xy is not None:
            xy = np.ascontiguousarray(xy, np.float32)
            xyp = _p(xy)
        self._check(lib().r3d_upload_regions(self._h, C.c_uint32(view_id), _p(desc), C.c_uint32(n), C.c_uint32(dim),
                                             C.c_int(dt), xyp))

    def liop_describe(self, image, keypoints, kp_size_factor=8.0):
        """image (h, w) float32; keypoints (n, 4) = x, y, size (diameter), angle (degrees) -> (n, 144) float32."""
        image = np.ascontiguousarray(image, np.float32)
        kps = np.ascontiguousarray(keypoints, np.float32).reshape(-1, 4)
        desc = np.zeros((len(kps), 144), np.float32)
        self._check(lib().r3d_liop_describe(self._h, _p(image), C.c_uint32(image.shape[1]), C.c_uint32(image.shape[0]),
                                            _p(kps), C.c_uint32(len(kps)), C.c_float(kp_size_factor), _p(desc)))
        return desc

    def akaze_detect(self, images, detector=DETECTOR_FAST_AKAZE, **opts):
        """Keypoints of a list of (h, w) float32 gray images in [0, 1] by Fast-AKAZE (the default) or, with
        detector=DETECTOR_AKAZE, by OpenCV's AKAZE: one akaze_keypoint_dtype array per image, in upstream order."""
        imgs = [np.ascontiguousarray(im, np.float32) for im in images]
        n = len(imgs)
        ptrs = (C.c_void_p * max(n, 1))(*[im.ctypes.data for im in imgs])
        ws = np.array([im.shape[1] if im.ndim == 2 else 0 for im in imgs] or [0], np.uint32)
        hs = np.array([im.shape[0] if im.ndim == 2 else 0 for im in imgs] or [0], np.uint32)
        f = C.c_void_p()
        self._check(lib().r3d_detect_keypoints(self._h, C.c_int(detector), ptrs, _p(ws), _p(hs), C.c_uint32(n),
                                               C.byref(akaze_options(**opts)), C.byref(f)))
        try:
            out = []
            for i in range(n):
                k = lib().r3d_features_count(f, C.c_uint32(i))
                a = np.zeros(k, akaze_keypoint_dtype)
                if k:
                    C.memmove(a.ctypes.data, lib().r3d_features_get(f, C.c_uint32(i)), k * akaze_keypoint_dtype.itemsize)
                out.append(a)
            return out
        finally:
            lib().r3d_free_features(f)

    def extract_features(self, images, out_dir=None, basenames=None, threshold=1e-3, kp_size_factor=8.0, progress=None,
                         detector=DETECTOR_FAST_AKAZE):
        """Keypoints (Fast-AKAZE by default, or detector=DETECTOR_AKAZE) described with LIOP-144, each image uploaded
        once: one (akaze_keypoint_dtype array,
        (n, 144) float32) pair per image.  out_dir: also write <out_dir>/<basenames[i]>.feat / .desc; progress(fraction,
        message, user), as compute_matches takes it, runs after each finished image (0.2 + 0.4 done / n)."""
        imgs = [np.ascontiguousarray(im, np.float32) for im in images]
        n = len(imgs)
        ptrs = (C.c_void_p * max(n, 1))(*[im.ctypes.data for im in imgs])
        ws = np.array([im.shape[1] if im.ndim == 2 else 0 for im in imgs] or [0], np.uint32)
        hs = np.array([im.shape[0] if im.ndim == 2 else 0 for im in imgs] or [0], np.uint32)
        o = ExtractOptions()
        lib().r3d_extract_default_options(C.byref(o))
        o.akaze = akaze_options(threshold=threshold)
        o.kp_size_factor = kp_size_factor
        names = None
        if out_dir is not None:
            o.out_dir = os.fsencode(out_dir)
        if basenames is not None:
            names = (C.c_char_p * max(len(basenames), 1))(*[None if b is None else os.fsencode(b) for b in basenames])
            o.basenames = C.cast(names, C.POINTER(C.c_char_p))
        cb = PROGRESS_CB(progress) if progress else C.cast(None, PROGRESS_CB)
        f = C.c_void_p()
        self._check(lib().r3d_extract_features_detector(self._h, C.c_int(detector), ptrs, _p(ws), _p(hs), C.c_uint32(n),
                                                        C.byref(o), cb, None, C.byref(f)))
        try:
            out = []
            for i in range(n):
                k = lib().r3d_features_count(f, C.c_uint32(i))
                a = np.zeros(k, akaze_keypoint_dtype)
                d = np.zeros((k, 144), np.float32)
                if k:
                    C.memmove(a.ctypes.data, lib().r3d_features_get(f, C.c_uint32(i)), k * akaze_keypoint_dtype.itemsize)
                    C.memmove(d.ctypes.data, lib().r3d_features_descriptors(f, C.c_uint32(i)), d.nbytes)
                out.append((a, d))
            return out
        finally:
            lib().r3d_free_features(f)

    def extract_timing(self):
        t = ExtractTiming()
        self._check(lib().r3d_get_extract_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in ExtractTiming._fields_}

    def akaze_timing(self):
        t = AkazeTiming()
        self._check(lib().r3d_get_akaze_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in AkazeTiming._fields_}

    def debug_akaze_refine(self, ldet, ratio, keypoints):
        """The refinement kernel alone on points (akaze_keypoint_dtype) of one level's Ldet; rejected: class_id -1."""
        ldet = np.ascontiguousarray(ldet, np.float32)
        kps = np.ascontiguousarray(keypoints, akaze_keypoint_dtype)
        out = np.zeros_like(kps)
        self._check(lib().r3d_debug_akaze_refine(self._h, _p(ldet), C.c_uint32(ldet.shape[1]), C.c_uint32(ldet.shape[0]),
                                                 C.c_float(ratio), _p(kps), C.c_uint32(len(kps)), _p(out)))
        return out

    def debug_akaze_levels(self, image, **opts):
        """One image through the detector's kernels: per level a dict with the level record, kcontrast, the five
        arrays (AKAZE_ARRAYS), the candidates after the same-level pass and their deletion flags after the lower- and
        the upper-level pass."""
        image = np.ascontiguousarray(image, np.float32)
        h, w = image.shape
        lv = akaze_levels(w, h, **{k: v for k, v in opts.items() if k != "threshold"})
        npx = sum(int(l["width"]) * int(l["height"]) for l in lv)
        cap = sum((int(l["width"]) + 1) // 2 * ((int(l["height"]) + 1) // 2) for l in lv)
        arrays = np.zeros(5 * npx, np.float32)
        kc = np.zeros(max(len(lv), 1), np.float32)
        cands = np.zeros(max(cap, 1), akaze_keypoint_dtype)
        flags = np.zeros(max(cap, 1), np.uint8)
        counts = np.zeros(max(len(lv), 1), np.uint32)
        self._check(lib().r3d_debug_akaze_levels(self._h, _p(image), C.c_uint32(w), C.c_uint32(h),
                                                 C.byref(akaze_options(**opts)), _p(arrays), _p(kc), _p(cands), _p(flags),
                                                 C.c_uint32(cap), _p(counts)))
        out, a, c = [], 0, 0
        for i, l in enumerate(lv):
            lw, lh = int(l["width"]), int(l["height"])
            d = {"level": l, "kcontrast": float(kc[i])}
            for name in AKAZE_ARRAYS:
                d[name] = arrays[a:a + lw * lh].reshape(lh, lw)
                a += lw * lh
            n = int(counts[i])
            d["candidates"] = cands[c:c + n].copy()
            d["deleted_lower"] = (flags[c:c + n] & 1).astype(bool)
            d["deleted_upper"] = (flags[c:c + n] & 2).astype(bool)
            c += n
            out.append(d)
        return out

    def debug_akaze_masks(self, image, **opts):
        """One image through the AKAZE detector's kernels: per level a dict with the level record, kcontrast, the five
        arrays (AKAZE_ARRAYS) and the kept-point masks (bool, level shape) after the same-level, the lower-level and
        the upper-level passes ("same", "lower", "upper")."""
        image = np.ascontiguousarray(image, np.float32)
        h, w = image.shape
        lv = akaze_levels(w, h, **{k: v for k, v in opts.items() if k != "threshold"})
        npx = sum(int(l["width"]) * int(l["height"]) for l in lv)
        arrays = np.zeros(max(5 * npx, 1), np.float32)
        kc = np.zeros(max(len(lv), 1), np.float32)
        masks = np.zeros(max(3 * npx, 1), np.uint8)
        self._check(lib().r3d_debug_akaze_masks(self._h, _p(image), C.c_uint32(w), C.c_uint32(h),
                                                C.byref(akaze_options(**opts)), _p(arrays), _p(kc), _p(masks)))
        out, a, m = [], 0, 0
        for i, l in enumerate(lv):
            lw, lh = int(l["width"]), int(l["height"])
            d = {"level": l, "kcontrast": float(kc[i])}
            for name in AKAZE_ARRAYS:
                d[name] = arrays[a:a + lw * lh].reshape(lh, lw)
                a += lw * lh
            for name in ("same", "lower", "upper"):
                d[name] = masks[m:m + lw * lh].reshape(lh, lw).astype(bool)
                m += lw * lh
            out.append(d)
        return out

    def debug_liop_process(self, patches):
        patches = np.ascontiguousarray(patches, np.float32).reshape(-1, 41 * 41)
        desc = np.zeros((len(patches), 144), np.float32)
        self._check(lib().r3d_debug_liop_process(self._h, _p(patches), C.c_uint32(len(patches)), _p(desc)))
        return desc

    def clear_regions(self):
        self._check(lib().r3d_clear_regions(self._h))

    def match_pairs(self, pairs, dist_ratio, flags=MATCH_DEFAULT):
        pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        h = C.c_void_p()
        self._check(lib().r3d_match_pairs(self._h, _p(pairs), C.c_uint64(len(pairs)), C.c_float(dist_ratio),
                                          C.c_uint32(flags), C.byref(h)))
        return Matches(h)

    def cascade_prepare(self, view_ids):
        """Hash the given (uploaded) views under their common zero-mean descriptor (R3D_MATCH_CASCADE_HASHING jobs that
        span several match_pairs calls)."""
        v = np.ascontiguousarray(view_ids, np.uint32).ravel()
        self._check(lib().r3d_cascade_prepare(self._h, _p(v), C.c_uint32(len(v))))

    def debug_cascade_view(self, view_id, n, dim):
        words = (dim + 31) // 32
        code = np.zeros((n, words), np.uint32)
        bucket = np.zeros((n, 6), np.uint16)
        ofs = np.zeros((6, 1025), np.uint32)
        ids = np.zeros((6, max(n, 1)), np.uint32)
        self._check(lib().r3d_debug_cascade_view(self._h, C.c_uint32(view_id), _p(code), _p(bucket), _p(ofs), _p(ids)))
        return code, bucket, ofs, ids[:, :n]

    def search_neighbours(self, view_db, view_query, n_query):
        idx = np.zeros((n_query, 2), np.int32)
        dist = np.zeros((n_query, 2), np.float32)
        self._check(lib().r3d_search_neighbours(self._h, C.c_uint32(view_db), C.c_uint32(view_query), _p(idx), _p(dist)))
        return idx, dist

    def debug_candidate_keys(self, view_db, view_query, n_query):
        npad = (max(n_query, 1) + 255) // 256 * 256
        keys = np.zeros((npad, 8), np.uint32)
        eps = C.c_float()
        self._check(lib().r3d_debug_candidate_keys(self._h, C.c_uint32(view_db), C.c_uint32(view_query), _p(keys), C.byref(eps)))
        return keys, eps.value

    def debug_view_operands(self, view_id):
        """The view's fp16 operands as the next matching call prepares them: dict with opQ, opD (n_pad x kp float16,
        None when the view has none), stats (max ||a||^2, max ||fp16(a)||^2, max ||a - fp16(a)||^2, max |a_k|) and
        the device's norm-split exponent e0."""
        n_pad, kp, e0 = C.c_uint32(), C.c_uint32(), C.c_int()
        self._check(lib().r3d_debug_view_operands(self._h, C.c_uint32(view_id), C.byref(n_pad), C.byref(kp), None, None,
                                                  None, None))
        opQ = np.zeros((n_pad.value, kp.value), np.float16)
        opD = np.zeros((n_pad.value, kp.value), np.float16)
        stats = np.zeros(4, np.float32)
        self._check(lib().r3d_debug_view_operands(self._h, C.c_uint32(view_id), C.byref(n_pad), C.byref(kp), _p(opQ),
                                                  _p(opD), _p(stats), C.byref(e0)))
        return {"opQ": opQ if kp.value else None, "opD": opD if kp.value else None, "stats": stats, "e0": e0.value}

    def debug_cholesky(self, A, method=CHOL_DENSE, ft=None, grid=0):
        """r3d_debug_cholesky on A ((n+1) x n: the matrix, whose lower triangle is read, and b as row n).  Returns
        (L (n+1) x n with y = L^-1 b as row n, x = A^-1 b, Linv (ceil(n/32), 32, 32) or None for the envelope
        kernel, not_pd bool)."""
        A = np.ascontiguousarray(A, np.float64)
        if A.ndim != 2 or A.shape[0] != A.shape[1] + 1:
            raise ValueError("A must be (n+1) x n")
        n = A.shape[1]
        ftp = None
        if ft is not None:
            ft = np.ascontiguousarray(ft, np.int32).ravel()
            if len(ft) != (n + 32) // 32:  # the library reads one entry per row tile of rows 0..n
                raise ValueError("ft must hold ceil((n+1)/32) = %d entries, not %d" % ((n + 32) // 32, len(ft)))
            ftp = _p(ft)
        L = np.empty((n + 1, n))
        x = np.empty(n)
        Linv = np.empty(((n + 31) // 32, 32, 32)) if method == CHOL_DENSE else None
        bad = C.c_int()
        self._check(lib().r3d_debug_cholesky(self._h, C.c_int(method), C.c_int(n), _p(A), ftp, C.c_int(grid), _p(L), _p(x),
                                             None if Linv is None else _p(Linv), C.byref(bad)))
        return L, x, Linv, bool(bad.value)

    def debug_chol_solve3(self, A, Y, grid=0):
        """r3d_debug_chol_solve3: X = A^-1 Y for A n x n (lower triangle read) and Y n x 3."""
        A = np.ascontiguousarray(A, np.float64)
        Y = np.ascontiguousarray(Y, np.float64)
        n = A.shape[1]
        if A.shape != (n, n) or Y.shape != (n, 3):
            raise ValueError("A must be n x n and Y n x 3")
        X = np.empty((n, 3))
        self._check(lib().r3d_debug_chol_solve3(self._h, C.c_int(n), _p(A), _p(Y), C.c_int(grid), _p(X)))
        return X

    def debug_acransac_score(self, model, x1, x2, models, max_thr, logalpha0, K, x3=None, per_point=False):
        """r3d_debug_acransac_score: the AC-RANSAC kernel's tier-1 bounds and tier-2 NFA scan of `models` (n x 9, or n x 12
        for the internal resection model 3) on one pair.  Returns a dict: "score" (ac_score_dtype per model), "logc_n"
        (M + 2 floats: log10 C(M, k), then the table's error bound), "logc_k" (M + 1) and, with per_point, "lo", "hi",
        "e" (n x M: the tier-1 interval and the tier-2 residual of every point)."""
        x1 = np.ascontiguousarray(x1, np.float64).reshape(-1, 2)
        x2 = np.ascontiguousarray(x2, np.float64).reshape(-1, 2)
        M = len(x1)
        if x2.shape != (M, 2):
            raise ValueError("x1 and x2 must both be M x 2")
        ms = 12 if model == 3 else 9
        models = np.ascontiguousarray(models, np.float64).reshape(-1, ms)
        n = len(models)
        K = np.ascontiguousarray(np.broadcast_to(np.asarray(K, np.float64).ravel(), (6,)), np.float64)
        x3p = None
        if x3 is not None:
            x3 = np.ascontiguousarray(x3, np.float64).ravel()
            if len(x3) != M:
                raise ValueError("x3 must hold M entries")
            x3p = _p(x3)
        out = np.zeros(max(n, 1), ac_score_dtype)
        logc_n = np.zeros(M + 2, np.float32)
        logc_k = np.zeros(M + 1, np.float32)
        lo = hi = e = None
        if per_point:
            lo, hi, e = (np.zeros((n, M)) for _ in range(3))
        self._check(lib().r3d_debug_acransac_score(
            self._h, C.c_int(model), C.c_uint32(M), _p(x1), _p(x2), x3p, C.c_double(max_thr), C.c_double(logalpha0), _p(K),
            _p(models), C.c_uint32(n), _p(out), *(None if a is None else _p(a) for a in (lo, hi, e)), _p(logc_n), _p(logc_k)))
        r = {"score": out[:n], "logc_n": logc_n, "logc_k": logc_k}
        if per_point:
            r.update(lo=lo, hi=hi, e=e)
        return r

    def filter_pairs(self, putative, widths, heights, model=MODEL_F, precision_px=4.0, max_iter=2048, Ks=None):
        n = len(widths)
        views = make_views(widths, heights, Ks)
        h = C.c_void_p()
        self._check(lib().r3d_filter_pairs(self._h, C.c_int(model), C.c_double(precision_px), C.c_uint32(max_iter),
                                           putative.handle, views, C.c_uint32(n), C.byref(h)))
        return Matches(h)

    def relative_poses(self, matches, widths, heights, Ks, precision_px=2.5, max_iter=256, refine=True, **ba):
        """r3d_relative_poses: relative pose of every pair of `matches` (map order).  Ks: n_views x 3 (focal, ppx, ppy).
        ba: r3d_ba_options fields of the two-view refinement.  Returns (numpy array of relpose_dtype, Matches of the
        AC-RANSAC inliers of the OK pairs)."""
        views = make_views(widths, heights, Ks)
        o = RelposeOptions()
        lib().r3d_relpose_default_options(C.byref(o))
        o.precision_px = precision_px
        o.max_iter = max_iter
        o.refine = int(refine)
        for k, v in ba.items():
            setattr(o.ba, k, v)
        out = np.zeros(max(matches.num_pairs, 1), relpose_dtype)
        h = C.c_void_p()
        self._check(lib().r3d_relative_poses(self._h, matches.handle, views, C.c_uint32(len(widths)), C.byref(o), _p(out),
                                             C.byref(h)))
        return out[:matches.num_pairs].copy(), Matches(h)

    @staticmethod
    def _resection_options(precision_px, max_iter, refine, ba):
        o = ResectionOptions()
        lib().r3d_resection_default_options(C.byref(o))
        o.precision_px = precision_px
        o.max_iter = max_iter
        o.refine = int(refine)
        for k, v in ba.items():
            setattr(o.ba, k, v)
        return o

    def resect_views(self, views, X, x, precision_px=float("inf"), max_iter=4096, refine=True, **ba):
        """r3d_resect_views: absolute pose of every view of `views` (a ResectionView array, e.g. from resection_views)
        from its 2D-3D correspondences X (n x 3), x (n x 2, pixels).  ba: r3d_ba_options fields of the pose refinement.
        Returns (numpy array of resection_dtype, inlier offsets [n_views + 1], inlier indices into each view's
        correspondences, in AC-RANSAC's residual order)."""
        X = np.ascontiguousarray(X, np.float64).reshape(-1, 3)
        x = np.ascontiguousarray(x, np.float64).reshape(-1, 2)
        n = len(views)
        o = self._resection_options(precision_px, max_iter, refine, ba)
        out = np.zeros(max(n, 1), resection_dtype)
        inl = np.zeros(max(len(x), 1), np.uint32)
        ofs = np.zeros(n + 1, np.uint64)
        self._check(lib().r3d_resect_views(self._h, views, C.c_uint32(n), _p(X), _p(x), C.byref(o), _p(out), _p(inl), _p(ofs)))
        return out[:n].copy(), ofs, inl[:int(ofs[n])].copy()

    def sfm_resect_views(self, sd, view_ids=None, precision_px=float("inf"), max_iter=4096, refine=True, **ba):
        """r3d_sfm_resect_views: resect the listed views of the SfmData (None: every view without a pose) against its
        structure and store the poses of the OK ones.  Returns a numpy array of resection_dtype."""
        o = self._resection_options(precision_px, max_iter, refine, ba)
        ids = np.ascontiguousarray([] if view_ids is None else view_ids, np.uint32)
        cap = len(ids) if len(ids) else lib().r3d_sfm_num_views(sd.h)
        out = np.zeros(max(cap, 1), resection_dtype)
        n_out = C.c_uint32(0)
        self._check(lib().r3d_sfm_resect_views(self._h, sd.h, _p(ids) if len(ids) else None, C.c_uint32(len(ids)), C.byref(o),
                                               _p(out), C.byref(n_out)))
        return out[:n_out.value].copy()

    def resection_timing(self):
        t = ResectionTiming()
        self._check(lib().r3d_get_resection_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in ResectionTiming._fields_}

    def rotation_averaging(self, rel, n_views, refine=True, max_angular_error_deg=5.0, method=ROTAVG_L2, **lm):
        """r3d_rotation_averaging on the OK entries of `rel` (relpose_dtype, e.g. from relative_poses).  lm: r3d_ba_options
        fields of the refinement (huber_a > 0: Huber loss).  Returns (rotations (n_views, 3, 3), view_kept (n_views,)
        bool, edge_kept (len(rel),) bool, edge_support (len(rel),) uint32, summary dict)."""
        rel = np.ascontiguousarray(rel, relpose_dtype)
        o = RotavgOptions()
        lib().r3d_rotavg_default_options(C.byref(o))
        o.method = method
        o.max_angular_error_deg = max_angular_error_deg
        o.refine = int(refine)
        for k, v in lm.items():
            setattr(o.lm, k, v)
        rot = np.zeros((max(n_views, 1), 3, 3))
        vk = np.zeros(max(n_views, 1), np.uint8)
        ek = np.zeros(max(len(rel), 1), np.uint8)
        sup = np.zeros(max(len(rel), 1), np.uint32)
        s = RotavgSummary()
        self._check(lib().r3d_rotation_averaging(self._h, _p(rel), C.c_uint64(len(rel)), C.c_uint32(n_views), C.byref(o), _p(rot),
                                                 _p(vk), _p(ek), _p(sup), C.byref(s)))
        summ = {k: getattr(s, k) for k, _ in RotavgSummary._fields_}
        return rot[:n_views], vk[:n_views].astype(bool), ek[:len(rel)].astype(bool), sup[:len(rel)].copy(), summ

    def rotation_averaging_l1(self, rel, n_views, **options):
        """r3d_rotation_averaging_l1 (Regard3D's L1 rotation averaging) on the OK entries of `rel` (relpose_dtype).
        options: r3d_rotavg_l1_options fields (max_angular_error_deg, irls_sigma_deg, l1_max_iterations,
        irls_max_iterations, tolerance); the others keep their defaults.  Returns the 5-tuple of rotation_averaging with
        this method's summary dict."""
        rel = np.ascontiguousarray(rel, relpose_dtype)
        o = RotavgL1Options()
        lib().r3d_rotavg_l1_default_options(C.byref(o))
        for k, v in options.items():
            if k not in dict(RotavgL1Options._fields_):
                raise TypeError("unknown option %r" % k)
            setattr(o, k, v)
        rot = np.zeros((max(n_views, 1), 3, 3))
        vk = np.zeros(max(n_views, 1), np.uint8)
        ek = np.zeros(max(len(rel), 1), np.uint8)
        sup = np.zeros(max(len(rel), 1), np.uint32)
        s = RotavgL1Summary()
        self._check(lib().r3d_rotation_averaging_l1(self._h, _p(rel), C.c_uint64(len(rel)), C.c_uint32(n_views), C.byref(o),
                                                    _p(rot), _p(vk), _p(ek), _p(sup), C.byref(s)))
        summ = {k: getattr(s, k) for k, _ in RotavgL1Summary._fields_}
        return rot[:n_views], vk[:n_views].astype(bool), ek[:len(rel)].astype(bool), sup[:len(rel)].copy(), summ

    def debug_rotavg_l1_step(self, rel, n_views, kind=0, rotations=None, state=None, tau=0.0, weights=None, rhs=None,
                             **options):
        """r3d_debug_rotavg_l1_step: one step of rotation_averaging_l1 on the same kept component (m views, E edges,
        n = m - 1).  kind 0: one primal-dual Newton iteration from state = (x, Ax, u, l1, l2, Atv) at tau, or with None
        from the start point; kind 1: one IRLS iteration; kind 2: the weighted normal equations for each row of weights /
        rhs ((K, 3E) each).  rotations: (n_views, 3, 3) by view id, None for the spanning-tree start.  options:
        r3d_rotavg_l1_options fields.  Returns a dict: m, E, n, view_ids, ab (E, 2), Rk (E, 3, 3), rotations0 (m, 3, 3),
        b (3E), cost (E), bmax, b_zero; kind 0: state0 / state (tuples as state; x and Atv (3n) component-major, the others
        3E), sdg0, tau0, resnorm0, sigx, rrow, w2, not_pd, laplacians (3, n + 1, n), dx, Adx, du, dl1, dl2, Atdv, rmin,
        step_max, trials ((step, residual norm) per trial), accepted, sdg, tau, resnorm; kind 1: w, wb, laplacians,
        not_pd, dx; kinds 0 and 1: rotations (m, 3, 3) after the update, xmax; kind 2: laplacians (K, 3, n + 1, n), dx
        (K, 3n; NaN for a system that is not positive definite), sys_not_pd (K)."""
        rel = np.ascontiguousarray(rel, relpose_dtype)
        o = RotavgL1Options()
        lib().r3d_rotavg_l1_default_options(C.byref(o))
        for k, v in options.items():
            if k not in dict(RotavgL1Options._fields_):
                raise TypeError("unknown option %r" % k)
            setattr(o, k, v)
        rot = None
        if rotations is not None:
            rot = np.ascontiguousarray(np.asarray(rotations, np.float64).reshape(-1, 9))
            if len(rot) < n_views:
                raise ValueError("rotations hold fewer than n_views views")
        x = None if state is None else np.ascontiguousarray(np.concatenate([np.asarray(a, np.float64).ravel() for a in state]))
        K = 1
        wt = rh = None
        if kind == 2:
            wt = np.ascontiguousarray(np.atleast_2d(np.asarray(weights, np.float64)))
            rh = np.ascontiguousarray(np.atleast_2d(np.asarray(rhs, np.float64)))
            if wt.shape != rh.shape:
                raise ValueError("weights and rhs must have the same shape")
            K = len(wt)
        mc, ec = max(n_views, 1), max(len(rel), 1)
        nr, nv, nst = 3 * ec, 3 * mc, 12 * ec + 6 * mc
        r = {"view_ids": np.zeros(mc, np.uint32), "ab": np.zeros(2 * ec, np.uint32), "Rk": np.zeros(9 * ec),
             "rotations0": np.zeros(9 * mc), "b": np.zeros(nr), "cost": np.zeros(ec), "state0": np.zeros(nst),
             "laplacians": np.zeros(K * 3 * mc * mc), "dx": np.full(K * nv, np.nan), "Atdv": np.zeros(nv), "rmin": np.zeros(ec),
             "state": np.zeros(nst), "rotations": np.zeros(9 * mc), "sys_not_pd": np.zeros(K, np.int32)}
        for k in ("sigx", "rrow", "w2", "Adx", "du", "dl1", "dl2", "w", "wb"):
            r[k] = np.zeros(nr)
        out = RotavgL1StepOut(**{k: v.ctypes.data for k, v in r.items()})
        self._check(lib().r3d_debug_rotavg_l1_step(self._h, _p(rel), C.c_uint64(len(rel)), C.c_uint32(n_views), C.byref(o),
                                                   None if rot is None else _p(rot), C.c_int(kind),
                                                   None if x is None else _p(x), C.c_uint64(0 if x is None else len(x)),
                                                   C.c_double(tau), None if wt is None else _p(wt), None if rh is None else _p(rh),
                                                   C.c_uint32(K), C.byref(out)))
        m, E = out.n_kept_views, out.n_kept_edges
        n = max(m, 1) - 1
        nr, nv = 3 * E, 3 * n

        def unpack(v):
            o1 = [0, nv, nv + nr, nv + 2 * nr, nv + 3 * nr, nv + 4 * nr, 2 * nv + 4 * nr]
            return tuple(v[o1[i]:o1[i + 1]].copy() for i in range(6))

        d = {"m": m, "E": E, "n": n, "view_ids": r["view_ids"][:m].copy(), "ab": r["ab"][:2 * E].reshape(E, 2).astype(np.int64),
             "Rk": r["Rk"][:9 * E].reshape(E, 3, 3).copy(), "rotations0": r["rotations0"][:9 * m].reshape(m, 3, 3).copy(),
             "b": r["b"][:nr].copy(), "cost": r["cost"][:E].copy(), "bmax": out.bmax, "b_zero": bool(out.b_zero),
             "not_pd": bool(out.not_pd), "rotations": r["rotations"][:9 * m].reshape(m, 3, 3).copy(), "xmax": out.xmax}
        lap = 3 * (n + 1) * n
        if kind == 2:
            d["laplacians"] = r["laplacians"][:K * lap].reshape(K, 3, n + 1, n).copy()
            d["dx"] = r["dx"][:K * nv].reshape(K, nv).copy()
            d["sys_not_pd"] = r["sys_not_pd"].astype(bool)
            return d
        d["laplacians"] = r["laplacians"][:lap].reshape(3, n + 1, n).copy()
        d["dx"] = r["dx"][:nv].copy()
        if kind == 1:
            d.update(w=r["w"][:nr].copy(), wb=r["wb"][:nr].copy())
            return d
        d.update(state0=unpack(r["state0"]), state=unpack(r["state"]), sdg0=out.sdg0, tau0=out.tau0, resnorm0=out.resnorm0,
                 step_max=out.step_max, trials=[(out.trial_step[t], out.trial_resnorm[t]) for t in range(out.n_trials)],
                 accepted=bool(out.accepted), sdg=out.sdg, tau=out.tau, resnorm=out.resnorm)
        for k in ("sigx", "rrow", "w2", "Adx", "du", "dl1", "dl2"):
            d[k] = r[k][:nr].copy()
        d.update(Atdv=r["Atdv"][:nv].copy(), rmin=r["rmin"][:E].copy())
        return d

    def translation_averaging(self, rel, rotations, rot_kept, n_views, method=TRANSAVG_L2_CHORDAL, edge_use=None,
                              softl1_loss=0.01, **lm):
        """r3d_translation_averaging on the OK entries of `rel` (relpose_dtype) with edge_use set (None: all of them, or
        rotation_averaging's edge_kept) and both views in rot_kept, given the global rotations (n_views, 3, 3) of
        rotation_averaging.  lm: r3d_ba_options fields (max_iterations / function_tolerance 0: the method's).  Returns
        (centers (n_views, 3), translations (n_views, 3), view_kept (n_views,) bool, edge_kept (len(rel),) bool,
        summary dict)."""
        rel = np.ascontiguousarray(rel, relpose_dtype)
        rot = np.ascontiguousarray(np.asarray(rotations, np.float64).reshape(-1, 3, 3))
        rk = np.ascontiguousarray(np.asarray(rot_kept).astype(np.uint8).ravel())
        if len(rot) < n_views or len(rk) < n_views:
            raise ValueError("rotations / rot_kept hold fewer than n_views views")
        use = None
        if edge_use is not None:
            use = np.ascontiguousarray(np.asarray(edge_use).astype(np.uint8).ravel())
            if len(use) != len(rel):
                raise ValueError("edge_use must have one entry per record")
        o = TransavgOptions()
        lib().r3d_transavg_default_options(C.byref(o))
        o.method = method
        o.softl1_loss = softl1_loss
        for k, v in lm.items():
            setattr(o.lm, k, v)
        cen = np.zeros((max(n_views, 1), 3))
        tra = np.zeros((max(n_views, 1), 3))
        vk = np.zeros(max(n_views, 1), np.uint8)
        ek = np.zeros(max(len(rel), 1), np.uint8)
        s = TransavgSummary()
        self._check(lib().r3d_translation_averaging(self._h, _p(rel), C.c_uint64(len(rel)), None if use is None else _p(use), _p(rot),
                                                    _p(rk), C.c_uint32(n_views), C.byref(o), _p(cen), _p(tra), _p(vk), _p(ek),
                                                    C.byref(s)))
        summ = {k: getattr(s, k) for k, _ in TransavgSummary._fields_}
        return cen[:n_views], tra[:n_views], vk[:n_views].astype(bool), ek[:len(rel)].astype(bool), summ

    def translation_averaging_l1(self, rel, rotations, rot_kept, n_views, edge_use=None, max_iterations=100, tolerance=1e-9):
        """r3d_translation_averaging_l1: the L-infinity translation LP (Regard3D's default L1 method) on the same edges as
        translation_averaging.  Returns (centers (n_views, 3), translations (n_views, 3), view_kept (n_views,) bool,
        edge_kept (len(rel),) bool, edge_scale (len(rel),) (lambda of the kept edges, 0 elsewhere), summary dict)."""
        rel = np.ascontiguousarray(rel, relpose_dtype)
        rot = np.ascontiguousarray(np.asarray(rotations, np.float64).reshape(-1, 3, 3))
        rk = np.ascontiguousarray(np.asarray(rot_kept).astype(np.uint8).ravel())
        if len(rot) < n_views or len(rk) < n_views:
            raise ValueError("rotations / rot_kept hold fewer than n_views views")
        use = None
        if edge_use is not None:
            use = np.ascontiguousarray(np.asarray(edge_use).astype(np.uint8).ravel())
            if len(use) != len(rel):
                raise ValueError("edge_use must have one entry per record")
        o = TransavgL1Options()
        lib().r3d_transavg_l1_default_options(C.byref(o))
        o.max_iterations = max_iterations
        o.tolerance = tolerance
        cen = np.zeros((max(n_views, 1), 3))
        tra = np.zeros((max(n_views, 1), 3))
        vk = np.zeros(max(n_views, 1), np.uint8)
        ek = np.zeros(max(len(rel), 1), np.uint8)
        lam = np.zeros(max(len(rel), 1))
        s = TransavgL1Summary()
        self._check(lib().r3d_translation_averaging_l1(self._h, _p(rel), C.c_uint64(len(rel)), None if use is None else _p(use),
                                                       _p(rot), _p(rk), C.c_uint32(n_views), C.byref(o), _p(cen), _p(tra), _p(vk),
                                                       _p(ek), _p(lam), C.byref(s)))
        summ = {k: getattr(s, k) for k, _ in TransavgL1Summary._fields_}
        return cen[:n_views], tra[:n_views], vk[:n_views].astype(bool), ek[:len(rel)].astype(bool), lam[:len(rel)].copy(), summ

    def debug_transavg_l1_step(self, rel, rotations, rot_kept, n_views, edge_use=None, state=None, tolerance=1e-9):
        """r3d_debug_transavg_l1_step: one iteration of translation_averaging_l1 on the same kept edges, from state =
        (y, lam, s, z) (y: T of the free kept views then gamma; lam, s, z in kept-edge order) or, with None, the
        solver's start point.  Returns a dict: m, ne, N, view_ids, edge_record, edge_ij (ne, 2), Rij (ne, 3, 3), u (ne, 3),
        state0 and state (each a (y, lam, s, z) tuple), norms (5), A ((N + 1) x N: the unscaled reduced matrix, row N
        the predictor's right-hand side), sc, not_pd (per attempt), retries, pred / corr dicts of dy, dlam, ds, dz,
        alpha_p, alpha_d (pred also complementarity, corr also rhs, scaled), sigma, converged, failed."""
        rel = np.ascontiguousarray(rel, relpose_dtype)
        rot = np.ascontiguousarray(np.asarray(rotations, np.float64).reshape(-1, 3, 3))
        rk = np.ascontiguousarray(np.asarray(rot_kept).astype(np.uint8).ravel())
        if len(rot) < n_views or len(rk) < n_views:
            raise ValueError("rotations / rot_kept hold fewer than n_views views")
        use = None
        if edge_use is not None:
            use = np.ascontiguousarray(np.asarray(edge_use).astype(np.uint8).ravel())
            if len(use) != len(rel):
                raise ValueError("edge_use must have one entry per record")
        x = None if state is None else np.ascontiguousarray(np.concatenate([np.asarray(a, np.float64).ravel() for a in state]))
        mc, ec = max(n_views, 1), max(len(rel), 1)
        nc = 3 * mc + 1
        nx = nc + 15 * ec
        r = {"view_ids": np.zeros(mc, np.uint32), "edge_record": np.zeros(ec, np.uint64), "edge_ij": np.zeros(2 * ec, np.uint32),
             "Rij": np.zeros(9 * ec), "u": np.zeros(3 * ec), "state0": np.zeros(nx), "A": np.zeros((nc + 1) * nc), "sc": np.zeros(nc),
             "corr_rhs": np.zeros(nc), "state": np.zeros(nx)}
        for ph in ("pred", "corr"):
            r.update({ph + "_dy": np.zeros(nc), ph + "_dlam": np.zeros(ec), ph + "_ds": np.zeros(7 * ec), ph + "_dz": np.zeros(7 * ec)})
        out = TransavgL1StepOut(**{k: v.ctypes.data for k, v in r.items()})
        self._check(lib().r3d_debug_transavg_l1_step(self._h, _p(rel), C.c_uint64(len(rel)), None if use is None else _p(use),
                                                     _p(rot), _p(rk), C.c_uint32(n_views), None if x is None else _p(x),
                                                     C.c_uint64(0 if x is None else len(x)), C.c_double(tolerance), C.byref(out)))
        m, ne, N = out.n_kept_views, out.n_kept_edges, out.n
        nr = 7 * ne

        def unpack(v):
            return v[:N].copy(), v[N:N + ne].copy(), v[N + ne:N + ne + nr].copy(), v[N + ne + nr:N + ne + 2 * nr].copy()

        d = {"m": m, "ne": ne, "N": N, "view_ids": r["view_ids"][:m].copy(), "edge_record": r["edge_record"][:ne].copy(),
             "edge_ij": r["edge_ij"][:2 * ne].reshape(ne, 2).copy(), "Rij": r["Rij"][:9 * ne].reshape(ne, 3, 3).copy(),
             "u": r["u"][:3 * ne].reshape(ne, 3).copy(), "state0": unpack(r["state0"]), "state": unpack(r["state"]),
             "norms": np.array(out.norms[:]), "A": r["A"][:(N + 1) * N].reshape(N + 1, N).copy(), "sc": r["sc"][:N].copy(),
             "not_pd": [bool(v) for v in out.not_pd], "retries": out.retries, "sigma": out.sigma,
             "converged": bool(out.converged), "failed": bool(out.failed)}
        for ph in ("pred", "corr"):
            d[ph] = {"dy": r[ph + "_dy"][:N].copy(), "dlam": r[ph + "_dlam"][:ne].copy(), "ds": r[ph + "_ds"][:nr].copy(),
                     "dz": r[ph + "_dz"][:nr].copy()}
        d["pred"].update(alpha_p=out.pred_alpha_p, alpha_d=out.pred_alpha_d, complementarity=out.pred_complementarity)
        d["corr"].update(alpha_p=out.alpha_p, alpha_d=out.alpha_d, rhs=r["corr_rhs"][:N].copy())
        return d

    def relpose_timing(self):
        t = RelposeTiming()
        self._check(lib().r3d_get_relpose_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in RelposeTiming._fields_}

    def match_timing(self):
        t = MatchTiming()
        self._check(lib().r3d_get_match_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in MatchTiming._fields_}

    def filter_timing(self):
        t = FilterTiming()
        self._check(lib().r3d_get_filter_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in FilterTiming._fields_}

    # ---- bundle adjustment ------------------------------------------------------------------
    @staticmethod
    def _ba_struct(p):
        s = BAProblem()
        s.n_cams = p["poses"].shape[0]
        s.n_pts = p["points"].shape[0]
        s.n_intr = p["intrinsics"].shape[0]
        s.n_obs = p["obs_xy"].shape[0]
        for k in ("poses", "intrinsics", "points", "obs_cam", "obs_pt", "cam_intr", "obs_xy"):
            setattr(s, k, p[k].ctypes.data)
        if p.get("intr_model") is not None:
            p["intr_model"] = np.ascontiguousarray(p["intr_model"], np.uint8)
            s.intr_model = p["intr_model"].ctypes.data
        if p.get("intrinsics_ext") is not None:
            p["intrinsics_ext"] = np.ascontiguousarray(p["intrinsics_ext"], np.float64)
            s.intrinsics_ext = p["intrinsics_ext"].ctypes.data
        if p.get("prior_cam") is not None and len(p["prior_cam"]):
            p["prior_cam"] = np.ascontiguousarray(p["prior_cam"], np.uint32)
            p["prior_center"] = np.ascontiguousarray(p["prior_center"], np.float64)
            p["prior_weight"] = np.ascontiguousarray(p["prior_weight"], np.float64)
            s.n_priors = len(p["prior_cam"])
            s.prior_cam = p["prior_cam"].ctypes.data
            s.prior_center = p["prior_center"].ctypes.data
            s.prior_weight = p["prior_weight"].ctypes.data
        return s

    def bundle_adjust(self, p, max_iterations=500, huber_a=16.0, refine_intrinsics=1, **tol):
        """In place on a dict of contiguous arrays (see synth.make_ba_problem / ba_prepare)."""
        o = BAOptions()
        lib().r3d_ba_default_options(C.byref(o))
        o.max_iterations = max_iterations
        o.huber_a = huber_a
        o.refine_intrinsics = refine_intrinsics
        for k, v in tol.items():
            setattr(o, k, v)
        s = self._ba_struct(p)
        summ = BASummary()
        trace = np.full(max_iterations + 1, np.nan, np.float64)
        self._check(lib().r3d_bundle_adjust(self._h, C.byref(s), C.byref(o), C.byref(summ), _p(trace)))
        d = {k: getattr(summ, k) for k, _ in BASummary._fields_}
        return d, trace[: summ.iterations + 1].copy()

    def debug_ba_step(self, p, radius, huber_a=16.0, refine_intrinsics=1, prior_huber_a=0.0, route=SCHUR_PLAN,
                      chol=CHOL_DENSE):
        """r3d_debug_ba_step: one LM step of bundle_adjust at p's parameters (p is not changed) and trust-region radius
        `radius`.  Returns a dict: g, diag, scale, delta (nparam = nB + 3 n_pts), S (nB x nB), rhs (nB), Vinv
        (n_pts x 3 x 3), and nB, n_batches, n_long, not_pd, gmax, model_cost_change, dx_norm2, x_norm2."""
        o = BAOptions()
        lib().r3d_ba_default_options(C.byref(o))
        o.huber_a, o.refine_intrinsics, o.prior_huber_a = huber_a, refine_intrinsics, prior_huber_a
        s = self._ba_struct(p)
        nB = 6 * s.n_cams + (6 * s.n_intr if refine_intrinsics else 0)
        nparam = nB + 3 * s.n_pts
        r = {k: np.empty(nparam) for k in ("g", "diag", "scale", "delta")}
        r["S"], r["rhs"], r["Vinv"] = np.empty((nB, nB)), np.empty(nB), np.empty((s.n_pts, 3, 3))
        out = BAStepOut(**{k: v.ctypes.data for k, v in r.items()})
        self._check(lib().r3d_debug_ba_step(self._h, C.byref(s), C.byref(o), C.c_double(radius), C.c_int(route), C.c_int(chol),
                                            C.byref(out)))
        for k in ("nB", "n_batches", "n_long", "gmax", "model_cost_change", "dx_norm2", "x_norm2"):
            r[k] = getattr(out, k)
        r["not_pd"] = bool(out.not_pd)
        return r

    # ---- multi-GPU bundle adjustment: one process per GPU, points partitioned (sharding.partition_ba) ----
    def comm_unique_id(self):
        """Rank 0 creates the id; the host distributes it (torch.distributed.broadcast_object_list, MPI, a file)."""
        buf = (C.c_uint8 * 128)()
        self._check(lib().r3d_comm_unique_id(self._h, buf))
        return bytes(buf)

    def comm_init(self, world, rank, comm_id):
        buf = (C.c_uint8 * 128).from_buffer_copy(comm_id)
        self._check(lib().r3d_comm_init(self._h, int(world), int(rank), buf))

    def comm_destroy(self):
        self._check(lib().r3d_comm_destroy(self._h))

    @property
    def comm_world(self):
        return int(lib().r3d_comm_world(self._h))

    def ba_residuals(self, p):
        s = self._ba_struct(p)
        res = np.zeros((p["obs_xy"].shape[0], 2), np.float64)
        self._check(lib().r3d_ba_residuals(self._h, C.byref(s), _p(res)))
        return res

    # ---- the steps either side of BA on an SfmData container (SURVEY.md 8f-3) --------------------------------
    def structure_from_tracks(self, sd, tracks):
        """Tracks -> landmarks of sd, triangulated from all posed views; returns the number of rejected tracks."""
        n = C.c_uint32()
        self._check(lib().r3d_sfm_structure_from_tracks(self._h, sd.h, tracks.h, C.byref(n)))
        return n.value

    def remove_outliers(self, sd, max_pixel_residual=4.0, min_track_length=2, min_angle_deg=2.0):
        a, b = C.c_uint32(), C.c_uint32()
        self._check(lib().r3d_sfm_remove_outliers(self._h, sd.h, C.c_double(max_pixel_residual), C.c_uint32(min_track_length),
                                                  C.c_double(min_angle_deg), C.byref(a), C.byref(b)))
        return a.value, b.value

    def colorize_plan(self, sd):
        """r3d_sfm_colorize_plan: (round_view[:n_rounds] view ids, lm_round (num_landmarks,) uint32,
        lm_pixel (num_landmarks, 2) int32 as (x, y)), landmarks in id order."""
        nv, nl = lib().r3d_sfm_num_views(sd.h), lib().r3d_sfm_num_landmarks(sd.h, 0)
        rv = np.zeros(max(nv, 1), np.uint32)
        nr = C.c_uint32()
        lr = np.zeros(max(nl, 1), np.uint32)
        lp = np.zeros((max(nl, 1), 2), np.int32)
        self._check(lib().r3d_sfm_colorize_plan(self._h, sd.h, _p(rv), C.byref(nr), _p(lr), _p(lp)))
        return rv[:nr.value].copy(), lr[:nl].copy(), lp[:nl].copy()

    def undistort_images(self, intrinsics, images):
        """UndistortImage with black fill of each H x W x 3 uint8 image through its intrinsic (a dict with model, focal,
        ppx, ppy, disto as SfmData.intrinsics() returns, or an SfmIntrinsic); returns the undistorted images.  The call's
        stage times are left in self.last_undistort_timing."""
        n = len(images)
        if len(intrinsics) != n:
            raise ValueError("one intrinsic per image")
        imgs = [np.ascontiguousarray(a, np.uint8) for a in images]
        for a in imgs:
            if a.ndim != 3 or a.shape[2] != 3:
                raise ValueError("images must be H x W x 3 uint8, got %s" % (a.shape,))
        intr = (SfmIntrinsic * max(n, 1))()
        for k, d in enumerate(intrinsics):
            if isinstance(d, SfmIntrinsic):
                intr[k] = d
                continue
            dist = list(d.get("disto", ())) + [0.0] * (5 - len(d.get("disto", ())))
            intr[k] = SfmIntrinsic(int(d.get("id", k)), int(d["model"]), int(d.get("width", 0)), int(d.get("height", 0)),
                                   float(d["focal"]), float(d["ppx"]), float(d["ppy"]), (C.c_double * 5)(*dist))
        outs = [np.empty_like(a) for a in imgs]
        src = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in imgs])
        dst = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in outs])
        ws = np.array([a.shape[1] for a in imgs] or [0], np.uint32)
        hs = np.array([a.shape[0] for a in imgs] or [0], np.uint32)
        t = UndistortTiming()
        self._check(lib().r3d_undistort_images(self._h, C.c_uint32(n), intr, src, _p(ws), _p(hs), dst, C.byref(t)))
        self.last_undistort_timing = {k: getattr(t, k) for k, _ in UndistortTiming._fields_}
        return outs

    def sfm_bundle_adjust(self, sd, max_iterations=500, refine_intrinsics=1, use_motion_priors=0, huber_a=16.0):
        class SfmBAOptions(C.Structure):
            _fields_ = [("solver", BAOptions), ("use_motion_priors", C.c_int)]
        o = SfmBAOptions()
        lib().r3d_sfm_ba_default_options(C.byref(o))
        o.solver.max_iterations = max_iterations
        o.solver.refine_intrinsics = refine_intrinsics
        o.solver.huber_a = huber_a
        o.use_motion_priors = use_motion_priors
        summ = BASummary()
        self._check(lib().r3d_sfm_bundle_adjust(self._h, sd.h, C.byref(o), C.byref(summ)))
        return {k: getattr(summ, k) for k, _ in BASummary._fields_}

    def compute_matches(self, matches_dir, basenames, widths, heights, dist_ratio=0.6, dim=144,
                        compute_fundamental=True, matching_algorithm=4, progress=None, f_filename=None,
                        compute_homography=False, compute_essential=False, Ks=None, svg_output=False):
        n = len(basenames)
        names = (C.c_char_p * n)(*[b.encode() for b in basenames])
        views = make_views(widths, heights, Ks)
        params = CMParams(dist_ratio, int(compute_fundamental), int(compute_essential), int(compute_homography),
                          matching_algorithm, dim, int(svg_output))
        paths = CMPaths(matches_dir.encode(), names, views, n, f_filename.encode() if f_filename else None, None, None)
        kp = (C.c_uint32 * n)()
        stats = CMStats()
        stats.n_views = n
        stats.number_of_keypoints = kp
        cb = PROGRESS_CB(progress) if progress else C.cast(None, PROGRESS_CB)
        self._check(lib().r3d_compute_matches(self._h, C.byref(params), C.byref(paths), cb, None, C.byref(stats)))
        d = {k: getattr(stats, k) for k, _ in CMStats._fields_ if k != "number_of_keypoints"}
        d["number_of_keypoints"] = [int(kp[k]) for k in range(n)]
        return d
