// sfm_structure.cu -- the steps either side of bundle adjustment (SURVEY.md 8f-3) on the SfM_Data container:
//   r3d_sfm_structure_from_tracks   tracks -> landmarks (observations from the uploaded feature positions), then
//                                   SfM_Data_Structure_Computation_Blind::triangulate: every landmark from all its posed
//                                   views (iteratively re-weighted DLT, openMVG `Triangulation::compute`), kept when the
//                                   smallest depth is positive
//   r3d_sfm_remove_outliers         RemoveOutliers_PixelResidualError + RemoveOutliers_AngleError (sfm_data_filters.hpp):
//                                   what the engines run after each bundle adjustment ("badTrackRejector")
// Upstream: OpenMVG 1.4 (un-vendored); driven by the engines at src/threads/R3DTriangulationThread.cpp:418-441, :492-512.
// One thread per landmark: the per-landmark work is a few hundred flops over <= a few hundred observations, the
// observation arrays are streamed once -- HBM-bound, no reuse to stage.
#include "r3d_internal.cuh"
#include "r3d_sfm.h"
#include "ba_model.cuh"
#include "p3p.cuh"

#include <cstring>

struct r3d_tracks {  // tracks.cpp
  std::vector<uint32_t> ids;
  std::vector<uint64_t> ofs;
  std::vector<uint32_t> views, feats;
};

namespace r3d {
namespace sfmk {

// K [R | t] of every camera (cam->get_projective_equivalent(pose)), row-major 3x4
__global__ void k_camera_matrices(const double* __restrict__ poses, const uint32_t* __restrict__ cam_intr,
                                  const double* __restrict__ intr, uint32_t n_cams, double* __restrict__ P) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cams) return;
  double R[9], Jr[9];
  ba::rotation_and_right_jacobian(poses + 6 * (size_t)c, R, Jr);
  const double* t = poses + 6 * (size_t)c + 3;
  const double* in = intr + 6 * (size_t)cam_intr[c];
  const double f = in[0], kx = in[1], ky = in[2];
  double* PM = P + 12 * (size_t)c;
  for (int j = 0; j < 3; ++j) {
    PM[j] = f * R[j] + kx * R[6 + j];
    PM[4 + j] = f * R[3 + j] + ky * R[6 + j];
    PM[8 + j] = R[6 + j];
  }
  PM[3] = f * t[0] + kx * t[2];
  PM[7] = f * t[1] + ky * t[2];
  PM[11] = t[2];
}

// cam->get_ud_pixel(x): radial K1 / K3 by bisection on the radius (as Pinhole_Intrinsic_Radial_K*::remove_disto), Brown
// T2 and fisheye by the resection step's Newton inverse (p3p::undistort_pixel), pinhole unchanged.
// in: f ppx ppy k1 k2 k3; ext: t1 t2 (Brown) or k4 (fisheye)
__device__ void undistort_pixel(int model, const double* in, const double* ext, double x, double y, double* ox, double* oy) {
  if (model == 4 || model == 5) {
    const double disto[5] = {in[3], in[4], in[5], ext[0], ext[1]};
    p3p::undistort_pixel(model, in[0], in[1], in[2], disto, x, y, ox, oy);
    return;
  }
  if (model < 2 || model > 3 || (in[3] == 0.0 && in[4] == 0.0 && in[5] == 0.0)) { *ox = x; *oy = y; return; }
  const double f = in[0], xd = (x - in[1]) / f, yd = (y - in[2]) / f;
  const double r2d = xd * xd + yd * yd;
  double s = 1.0;
  if (r2d != 0.0) {
    const double k1 = in[3], k2 = model == 3 ? in[4] : 0.0, k3 = model == 3 ? in[5] : 0.0;
    auto disto = [&](double r2) { const double c = 1.0 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2; return r2 * c * c; };
    double lo = r2d, hi = r2d;
    while (disto(lo) > r2d) lo /= 1.05;
    while (disto(hi) < r2d) hi *= 1.05;
    while (1e-8 < hi - lo) {
      const double mid = .5 * (lo + hi);
      if (disto(mid) > r2d) hi = mid; else lo = mid;
    }
    s = sqrt(.5 * (lo + hi) / r2d);
  }
  *ox = f * xd * s + in[1];
  *oy = f * yd * s + in[2];
}

// `Triangulation::compute(3)` per landmark; ok = at least two observations and a positive smallest depth
__global__ void __launch_bounds__(128) k_triangulate(uint32_t n_lm, const uint64_t* __restrict__ obs_ofs,
                                                     const uint32_t* __restrict__ obs_cam, const double2* __restrict__ obs_xy,
                                                     const double* __restrict__ P, const uint32_t* __restrict__ cam_intr,
                                                     const double* __restrict__ intr, const uint8_t* __restrict__ intr_model,
                                                     const double* __restrict__ intr_ext, double* __restrict__ X,
                                                     uint8_t* __restrict__ ok) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n_lm) return;
  const uint64_t b = obs_ofs[l], e = obs_ofs[l + 1];
  ok[l] = 0;
  if (e - b < 2) return;
  double Xl[3] = {0, 0, 0}, zmin = 0;
  for (int it = 0; it < 3; ++it) {
    double AtA[6] = {0, 0, 0, 0, 0, 0}, Atb[3] = {0, 0, 0};  // AtA: 00 10 11 20 21 22
    for (uint64_t o = b; o < e; ++o) {
      const uint32_t c = obs_cam[o], g = cam_intr[c];
      const double* PM = P + 12 * (size_t)c;
      double px, py;
      undistort_pixel(intr_model ? (int)intr_model[g] : 3, intr + 6 * (size_t)g, intr_ext + 2 * (size_t)g, obs_xy[o].x, obs_xy[o].y,
                      &px, &py);
      double w = 1.0;
      if (it > 0) w = 1.0 / (PM[8] * Xl[0] + PM[9] * Xl[1] + PM[10] * Xl[2] + PM[11]);
      double v1[3], v2[3];
      for (int j = 0; j < 3; ++j) {
        v1[j] = w * (PM[j] - px * PM[8 + j]);
        v2[j] = w * (PM[4 + j] - py * PM[8 + j]);
        Atb[j] += w * (v1[j] * (px * PM[11] - PM[3]) + v2[j] * (py * PM[11] - PM[7]));
      }
      AtA[0] += v1[0] * v1[0] + v2[0] * v2[0];
      AtA[1] += v1[1] * v1[0] + v2[1] * v2[0];
      AtA[2] += v1[1] * v1[1] + v2[1] * v2[1];
      AtA[3] += v1[2] * v1[0] + v2[2] * v2[0];
      AtA[4] += v1[2] * v1[1] + v2[2] * v2[1];
      AtA[5] += v1[2] * v1[2] + v2[2] * v2[2];
    }
    const double a[9] = {AtA[0], AtA[1], AtA[3], AtA[1], AtA[2], AtA[4], AtA[3], AtA[4], AtA[5]};
    const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
    const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
    const double inv[9] = {c00 / det, (a[2] * a[7] - a[1] * a[8]) / det, (a[1] * a[5] - a[2] * a[4]) / det,
                           c01 / det, (a[0] * a[8] - a[2] * a[6]) / det, (a[2] * a[3] - a[0] * a[5]) / det,
                           c02 / det, (a[1] * a[6] - a[0] * a[7]) / det, (a[0] * a[4] - a[1] * a[3]) / det};
    for (int i = 0; i < 3; ++i) Xl[i] = inv[3 * i] * Atb[0] + inv[3 * i + 1] * Atb[1] + inv[3 * i + 2] * Atb[2];
    zmin = 1.7976931348623157e308;
    for (uint64_t o = b; o < e; ++o) {
      const double* PM = P + 12 * (size_t)obs_cam[o];
      zmin = fmin(zmin, PM[8] * Xl[0] + PM[9] * Xl[1] + PM[10] * Xl[2] + PM[11]);
    }
  }
  X[3 * (size_t)l] = Xl[0]; X[3 * (size_t)l + 1] = Xl[1]; X[3 * (size_t)l + 2] = Xl[2];
  ok[l] = zmin > 0 ? 1 : 0;
}

// per landmark: which observations keep a pixel residual norm <= thr, and the largest angle between two of its rays
__global__ void __launch_bounds__(128) k_landmark_checks(uint32_t n_lm, const uint64_t* __restrict__ obs_ofs,
                                                         const uint32_t* __restrict__ obs_cam, const double2* __restrict__ obs_xy,
                                                         const double* __restrict__ poses, const uint32_t* __restrict__ cam_intr,
                                                         const double* __restrict__ intr, const uint8_t* __restrict__ intr_model,
                                                         const double* __restrict__ intr_ext, const double* __restrict__ X,
                                                         double thr_px, uint8_t* __restrict__ keep_obs, double* __restrict__ max_angle) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n_lm) return;
  const uint64_t b = obs_ofs[l], e = obs_ofs[l + 1];
  const double* Xl = X + 3 * (size_t)l;
  for (uint64_t o = b; o < e; ++o) {
    const uint32_t c = obs_cam[o], g = cam_intr[c];
    double r[2];
    ba::residual_only(intr_model ? (int)intr_model[g] : 3, intr + 6 * (size_t)g, intr_ext ? intr_ext + 2 * (size_t)g : nullptr,
                      poses + 6 * (size_t)c, Xl, obs_xy[o].x, obs_xy[o].y, r);
    keep_obs[o] = sqrt(r[0] * r[0] + r[1] * r[1]) > thr_px ? 0 : 1;
  }
  double best = 0.0;
  for (uint64_t a = b; a < e; ++a) {
    double Ra[9], Jr[9], u[3];
    const double* pa = poses + 6 * (size_t)obs_cam[a];
    ba::rotation_and_right_jacobian(pa, Ra, Jr);
    for (int i = 0; i < 3; ++i) u[i] = Xl[i] + (Ra[i] * pa[3] + Ra[3 + i] * pa[4] + Ra[6 + i] * pa[5]);  // X - C
    const double nu = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
    for (uint64_t q = a + 1; q < e; ++q) {
      double Rq[9], v[3];
      const double* pq = poses + 6 * (size_t)obs_cam[q];
      ba::rotation_and_right_jacobian(pq, Rq, Jr);
      for (int i = 0; i < 3; ++i) v[i] = Xl[i] + (Rq[i] * pq[3] + Rq[3 + i] * pq[4] + Rq[6 + i] * pq[5]);
      const double nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
      double cs = (u[0] * v[0] + u[1] * v[1] + u[2] * v[2]) / (nu * nv);
      cs = cs > 1.0 ? 1.0 : (cs < -1.0 ? -1.0 : cs);
      best = fmax(best, acos(cs) * (180.0 / 3.14159265358979323846));
    }
  }
  max_angle[l] = best;
}

}  // namespace sfmk
}  // namespace r3d

using namespace r3d;

namespace {

struct DevScene {
  DeviceWorker* w;
  std::vector<void*> blocks;
  double *poses = nullptr, *intr = nullptr, *ext = nullptr, *X = nullptr, *P = nullptr, *angle = nullptr;
  double2* obs_xy = nullptr;
  uint8_t *model = nullptr, *ok = nullptr, *keep = nullptr;
  uint32_t *cam_intr = nullptr, *obs_cam = nullptr;
  uint64_t* obs_ofs = nullptr;
  ~DevScene() { cudaStreamSynchronize(w->stream); for (void* p : blocks) pool_release(*w, p); }
  template <typename T>
  bool up(T** d, const void* h, size_t n) {
    *d = (T*)pool_alloc(*w, std::max<size_t>(n, 1) * sizeof(T));
    if (!*d) return false;
    blocks.push_back(*d);
    return !h || n == 0 || cudaMemcpyAsync(*d, h, n * sizeof(T), cudaMemcpyHostToDevice, w->stream) == cudaSuccess;
  }
};

int upload(r3d_ctx* ctx, const r3d_sfm::Flat& F, DevScene& D) {
  const size_t n_lm = F.lm_ids.size(), n_obs = F.obs_cam.size(), n_cams = F.pose_index.size();
  bool ok = D.up(&D.poses, F.poses.data(), F.poses.size()) && D.up(&D.intr, F.intr.data(), F.intr.size()) &&
            D.up(&D.ext, F.ext.data(), F.ext.size()) && D.up(&D.X, F.X.data(), F.X.size()) && D.up(&D.model, F.model.data(), F.model.size()) &&
            D.up(&D.cam_intr, F.cam_intr.data(), F.cam_intr.size()) && D.up(&D.obs_cam, F.obs_cam.data(), n_obs) &&
            D.up(&D.obs_xy, F.obs_xy.data(), n_obs) && D.up(&D.obs_ofs, F.obs_ofs.data(), F.obs_ofs.size()) &&
            D.up(&D.P, nullptr, 12 * n_cams) && D.up(&D.ok, nullptr, n_lm) && D.up(&D.keep, nullptr, n_obs) && D.up(&D.angle, nullptr, n_lm);
  if (!ok) return fail(ctx, R3D_ERR_NOMEM, "sfm structure: device allocation / upload failed");
  return R3D_OK;
}

}  // namespace

extern "C" int r3d_sfm_structure_from_tracks(r3d_ctx* ctx, r3d_sfm_data* sd, const r3d_tracks* tracks, uint32_t* n_rejected) try {
  if (!ctx || !sd || !tracks) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_structure_from_tracks: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  // tracks -> landmarks: observation = position of the feature in its view (uploaded with the regions)
  sd->structure.clear();
  for (size_t k = 0; k < tracks->ids.size(); ++k) {
    r3d_sfm_data::Landmark lm;
    lm.X[0] = lm.X[1] = lm.X[2] = 0.0;
    for (uint64_t q = tracks->ofs[k]; q < tracks->ofs[k + 1]; ++q) {
      const uint32_t v = tracks->views[q], f = tracks->feats[q];
      auto it = w.views.find(v);
      if (it == w.views.end() || !it->second.has_xy || f >= it->second.n)
        return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_structure_from_tracks: positions of a tracked feature were not uploaded");
      r3d_sfm_data::Obs ob;
      ob.id_feat = f;
      ob.x[0] = (double)it->second.h_xy[2 * (size_t)f];
      ob.x[1] = (double)it->second.h_xy[2 * (size_t)f + 1];
      lm.obs[v] = ob;
    }
    sd->structure[tracks->ids[k]] = std::move(lm);
  }
  r3d_sfm::Flat F;
  int rc = r3d_sfm::flatten(*sd, /*skip_undefined=*/true, F);
  if (rc) return fail(ctx, rc, "r3d_sfm_structure_from_tracks: a pose is shared by views with different intrinsics");
  uint32_t rejected = 0;
  const uint32_t n_lm = (uint32_t)F.lm_ids.size();
  if (n_lm && !F.pose_index.empty() && !F.intr_index.empty()) {
    DevScene D{&w, {}};
    if ((rc = upload(ctx, F, D))) return rc;
    const uint32_t n_cams = (uint32_t)F.pose_index.size();
    sfmk::k_camera_matrices<<<(n_cams + 127) / 128, 128, 0, w.stream>>>(D.poses, D.cam_intr, D.intr, n_cams, D.P);
    sfmk::k_triangulate<<<(n_lm + 127) / 128, 128, 0, w.stream>>>(n_lm, D.obs_ofs, D.obs_cam, D.obs_xy, D.P, D.cam_intr, D.intr, D.model, D.ext,
                                                                  D.X, D.ok);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    std::vector<uint8_t> hok(n_lm);
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(F.X.data(), D.X, F.X.size() * 8, cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hok.data(), D.ok, n_lm, cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    for (uint32_t l = 0; l < n_lm; ++l) {
      if (hok[l]) std::memcpy(sd->structure[F.lm_ids[l]].X, &F.X[3 * (size_t)l], 3 * sizeof(double));
      else { sd->structure.erase(F.lm_ids[l]); ++rejected; }  // "Erase the unsuccessful triangulated tracks"
    }
  } else {
    rejected = (uint32_t)sd->structure.size();
    sd->structure.clear();
  }
  if (n_rejected) *n_rejected = rejected;
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; }

extern "C" int r3d_sfm_remove_outliers(r3d_ctx* ctx, r3d_sfm_data* sd, double max_pixel_residual, uint32_t min_track_length,
                                       double min_angle_deg, uint32_t* removed_observations, uint32_t* removed_landmarks) try {
  if (!ctx || !sd) return fail(ctx, R3D_ERR_INVALID, "r3d_sfm_remove_outliers: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  r3d_sfm::Flat F;
  int rc = r3d_sfm::flatten(*sd, /*skip_undefined=*/true, F);
  if (rc) return fail(ctx, rc, "r3d_sfm_remove_outliers: a pose is shared by views with different intrinsics");
  uint32_t rm_obs = 0, rm_lm = 0;
  const uint32_t n_lm = (uint32_t)F.lm_ids.size();
  if (n_lm && !F.obs_cam.empty()) {
    DevScene D{&w, {}};
    if ((rc = upload(ctx, F, D))) return rc;
    sfmk::k_landmark_checks<<<(n_lm + 127) / 128, 128, 0, w.stream>>>(n_lm, D.obs_ofs, D.obs_cam, D.obs_xy, D.poses, D.cam_intr, D.intr,
                                                                      D.model, D.ext, D.X, max_pixel_residual, D.keep, D.angle);
    R3D_CUDA_TRY(ctx, cudaGetLastError());
    std::vector<uint8_t> keep(F.obs_cam.size());
    std::vector<double> angle(n_lm);
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(keep.data(), D.keep, keep.size(), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(angle.data(), D.angle, n_lm * 8, cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    for (uint32_t l = 0; l < n_lm; ++l) {
      auto it = sd->structure.find(F.lm_ids[l]);
      // RemoveOutliers_PixelResidualError: drop the observations beyond the threshold, then too short tracks
      for (uint64_t o = F.obs_ofs[l]; o < F.obs_ofs[l + 1]; ++o)
        if (!keep[o]) { it->second.obs.erase(F.obs_view[o]); ++rm_obs; }
      if (it->second.obs.empty() || it->second.obs.size() < min_track_length) { sd->structure.erase(it); ++rm_lm; continue; }
      // RemoveOutliers_AngleError: the largest angle between two rays must reach the minimum
      // (evaluated on the observation set BEFORE the residual pass; upstream runs the two filters back to back and the
      // second sees the pruned set -- recompute when something was dropped)
      bool dropped = false;
      for (uint64_t o = F.obs_ofs[l]; o < F.obs_ofs[l + 1]; ++o) dropped |= !keep[o];
      if (min_angle_deg > 0.0 && !dropped && angle[l] < min_angle_deg) { sd->structure.erase(it); ++rm_lm; }
    }
    if (min_angle_deg > 0.0 && rm_obs) {  // landmarks that lost observations: angle test on what is left (second pass)
      uint32_t more_obs = 0, more_lm = 0;
      rc = r3d_sfm_remove_outliers(ctx, sd, 1e300, 0, min_angle_deg, &more_obs, &more_lm);
      if (rc) return rc;
      rm_lm += more_lm;
    }
  }
  if (removed_observations) *removed_observations = rm_obs;
  if (removed_landmarks) *removed_landmarks = rm_lm;
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; }
