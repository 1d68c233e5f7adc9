// acransac.cuh -- shared declarations of the AC-RANSAC fundamental filter (host + device).
#pragma once
#include "r3d_internal.cuh"

namespace r3d {

struct AcPair {          // per image pair (device)
  uint32_t pt_ofs;       // first point of this pair in x1/x2
  uint32_t M;            // number of putative matches
  uint32_t tbl_ofs;      // first entry of this pair's logc_n table
  uint32_t pad_;
  double max_thr;        // precision^2 * N2(0,0)^2
  double logalpha0;      // F: log10(2 D / A / N2(0,0)) ; H: log10(pi / (w h) / N2(0,0)^2), image J
  double loge0;          // log10(MAX_MODELS * (M - MINIMUM_SAMPLES))
  double K[6];           // essential model: f, ppx, ppy of image I, then of image J (pinhole K)
                         // resection model: f, ppx, ppy of the view, then K[3] = the squared residual the tier-1
                         // histogram's top bin starts at (the precision may be infinite there)
};

// internal model ids: 0 = F (7-point), 1 = H (4-point), 2 = E (5-point), 3 = resection with known K (P3P: x1 holds
// X.xy, x3 holds X.z, x2 the undistorted pixel; the model is P = K [R | t], 3 x 4); Kernel::MINIMUM_SAMPLES / MAX_MODELS
__host__ __device__ constexpr uint32_t ac_min_samples(int model) {
  return model == 0 ? 7u : (model == 1 ? 4u : (model == 2 ? 5u : 3u));
}
__host__ __device__ constexpr uint32_t ac_max_models(int model) {
  return model == 0 ? 3u : (model == 1 ? 1u : (model == 2 ? 10u : 4u));
}
__host__ __device__ constexpr uint32_t ac_model_size(int model) { return model == 3 ? 12u : 9u; }  // doubles per model

struct AcPointSrc {      // per pair: where its matched positions come from and how they are normalised
  const float2* xyI;     // positions of view I / J on the device (uploaded with the regions)
  const float2* xyJ;
  double s1, c1x, c1y;   // x1 = s1 * x + c1  (ACKernelAdaptor normalisation; identity for the essential model)
  double s2, c2x, c2y;
  uint32_t nI, nJ, identity, pad_;
};

struct AcFusedOut {      // per pair, written by the persistent kernel (acransac_fused.cu)
  double minNFA, errorMax;
  uint32_t n_inliers;    // 0 when minNFA >= 0; else the best model's inliers, listed in residual order
  uint32_t iterations;   // RANSAC iterations the state machine consumed
  uint32_t exact_scores; // models that needed the sort + exact NFA scan (tier 2)
  uint32_t models;       // models scored
  uint32_t events;       // pool replacements
  uint32_t pad_;
};

// persistent one-CTA-per-pair ACRANSAC (acransac_fused.cu); `order`: pair ids of one size class, largest first;
// huge: sort buffers / pool in global scratch (cap entries per CTA of the grid); out_model (may be null):
// ac_model_size(model) doubles per pair id, the best model of every pair with inliers (F = K2^-T E K1^-1 for the
// essential model); x3: the resection model's third point coordinate, null for the others
size_t acransac_fused_smem_bytes(int model, uint32_t cap, bool huge);
int acransac_fused_ctas_per_sm(int model, uint32_t cap, bool huge);
int launch_acransac_fused(r3d_ctx* ctx, DeviceWorker& w, int model, bool huge, const AcPair* pairs, const uint32_t* order,
                          uint32_t n_order, uint32_t* work_counter, const double2* x1, const double2* x2, const float* logc_n,
                          const float* logc_k, uint32_t cap, uint32_t max_iter, double* g_se, uint32_t* g_si, uint32_t* g_pool,
                          const uint2* matches, uint2* out_matches, AcFusedOut* out, double* out_model, uint32_t grid,
                          const double* x3 = nullptr);

// The one driver of k_acransac_fused, shared by the filters (run_fused) and resection (resect_range), in two steps so
// that each caller times the launches alone (acransac_host.cu).  plan(): cuts the problems into size classes
// (shared-memory sort capacity 1024 ... 16384 matches; beyond that the "huge" class sorts in global scratch), largest
// first within a class, sizes the grid of every class, allocates the scratch and uploads the launch order;
// R3D_ERR_UNSUPPORTED when the device sample stream disagrees with this process's <random> (rng_selftest).  launch():
// one persistent launch per class, the huge class first, adding them to `launches`; no synchronisation.  The object
// owns the scratch the launches use: the caller keeps it until it has synchronised w.stream.
struct AcFused {
  static constexpr int kClasses = 6;  // caps 1024, 2048, 4096, 8192, 16384, huge
  int model = 0;
  uint32_t class_ofs[kClasses + 1] = {}, caps[kClasses] = {}, grids[kClasses] = {};
  std::vector<uint32_t> horder;       // problem ids, class after class
  DevArr<uint32_t> order, work, si, pool;
  DevArr<double> se;
  explicit AcFused(DeviceWorker& w) : order(w), work(w), si(w), pool(w), se(w) {}
  int plan(r3d_ctx* ctx, DeviceWorker& w, int model, const std::vector<AcPair>& pairs);
  int launch(r3d_ctx* ctx, DeviceWorker& w, const AcPair* d_pairs, const double2* x1, const double2* x2, const double* x3,
             const float* logc_n, const float* logc_k, uint32_t max_iter, const uint2* matches, uint2* out_matches,
             AcFusedOut* out, double* out_model, uint64_t& launches);
};

// The log-combinatorial tables of a batch of problems (acransac_host.cu).  upload(): the log10 table k = 0 .. maxM + 1
// (single precision, as upstream's makelogcombi builds it) and logc_k = makelogcombi_k, log10 C(n, ns) for n = 0 .. maxM
// (the running float sum upstream builds), copied to the device; logc_n sized to tbl_total entries, for
// launch_ac_tables to fill from vlog10.
struct AcTables {
  std::vector<float> h_vlog10, h_logc_k;
  DevArr<float> vlog10, logc_n, logc_k;
  explicit AcTables(DeviceWorker& w) : vlog10(w), logc_n(w), logc_k(w) {}
  int upload(r3d_ctx* ctx, DeviceWorker& w, uint32_t ns, uint32_t maxM, uint64_t tbl_total);
};

// r3d_debug_acransac_score on one pair already on the device (acransac_fused.cu): d_pair->pt_ofs = tbl_ofs = 0,
// d_se / d_si: debug_acransac_cap(M) entries, d_lo / d_hi / d_e: n_models x M or null
uint32_t debug_acransac_cap(uint32_t M);
int debug_acransac_score(r3d_ctx* ctx, DeviceWorker& w, int model, const AcPair* d_pair, const double2* d_x1, const double2* d_x2,
                         const double* d_x3, const float* d_logc_n, const float* d_logc_k, const double* d_models, uint32_t n_models,
                         uint32_t M, double* d_se, uint32_t* d_si, r3d_ac_score* d_out, double* d_lo, double* d_hi, double* d_e);

struct AcBestModel {      // per pair of the putative map (r3d_relative_poses): the kept pair's best model, errorMax
  double model[9];       // row-major; F = K2^-T E K1^-1 for the essential model
  double errorMax;       // squared residual of the last inlier
};
// AC-RANSAC of the pairs [p0, p1) of a putative map on one worker (acransac_host.cu); result[p]: inliers of pair p.
// best (may be null): the best model and errorMax of every kept pair
int filter_pairs_model(r3d_ctx* ctx, DeviceWorker& w, int model, double precision_px, uint32_t max_iter, const r3d_matches* put,
                       const r3d_view_info* views, uint32_t n_views, uint64_t p0, uint64_t p1, r3d_filter_timing& T,
                       std::vector<std::vector<r3d_indmatch>>& result, std::vector<AcBestModel>* best = nullptr);

// x1/x2[pt_ofs + k] = normalised positions of putative match k of every pair (double, like MatchesPairToMat)
int launch_ac_points(r3d_ctx* ctx, DeviceWorker& w, const AcPair* pairs, const AcPointSrc* src, uint32_t n_pairs,
                     const uint2* matches, double2* x1, double2* x2, uint32_t* bad_flag);
int launch_ac_tables(r3d_ctx* ctx, DeviceWorker& w, const AcPair* pairs, uint32_t n_pairs, const float* vlog10, float* logc_n);

}  // namespace r3d
