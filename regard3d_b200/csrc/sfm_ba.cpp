// sfm_ba.cpp -- openMVG::sfm::Bundle_Adjustment_Ceres::Adjust(SfM_Data&, Optimize_Options) on the library's SfM_Data
// container: r3d_sfm::flatten (sfm_scene.cpp) -> r3d_bundle_adjust (ba.cu) -> write back.  This is what the SfM engines
// call between their resection / triangulation rounds (src/threads/R3DTriangulationThread.cpp:441, :512, :250 ->
// engine.Process()); the C++ adaptor with the reference's class name is regard3d_b200/csrc/Bundle_Adjustment_b200.h.
//
// Parameterisation as in OpenMVG's BA (SURVEY.md A.7): pose = angle-axis(R) | t with t = -R C (Pose3 stores R and the
// centre C); one parameter block per intrinsic id (params in getParams() order), one per landmark.  Options mapped:
// intrinsics ADJUST_ALL / NONE (the two the reference uses, R3DTriangulationThread.cpp:429-432), extrinsics and
// structure ADJUST_ALL, control points unused, use_motion_priors -> one pose-centre block per ViewPriors view.  NOT
// restated: the robust similarity registration of the scene to the GPS frame that OpenMVG runs before adding the prior
// blocks (it needs >= 3 priors and changes the gauge, not the reprojection cost); pass prior_huber_a = the fitting error
// of your own registration, or 0 for a quadratic prior.
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "r3d_sfm.h"

extern "C" void r3d_sfm_ba_default_options(r3d_sfm_ba_options* o) {
  if (!o) return;
  r3d_ba_default_options(&o->solver);
  o->use_motion_priors = 0;
}

extern "C" int r3d_sfm_bundle_adjust(r3d_ctx* ctx, r3d_sfm_data* sd, const r3d_sfm_ba_options* opt, r3d_ba_summary* summary) try {
  if (!ctx || !sd || !opt || !summary) return R3D_ERR_INVALID;
  r3d_sfm::Flat F;
  const int frc = r3d_sfm::flatten(*sd, /*skip_undefined=*/false, F);  // upstream, map::at throws on an undefined view
  if (frc) return frc;
  if (F.intr_index.empty() || F.pose_index.empty() || F.lm_ids.empty()) return R3D_ERR_INVALID;
  std::vector<uint32_t> obs_pt(F.obs_cam.size());
  for (uint32_t l = 0; l < F.lm_ids.size(); ++l) std::fill(obs_pt.begin() + F.obs_ofs[l], obs_pt.begin() + F.obs_ofs[l + 1], l);
  std::vector<uint32_t> prior_cam;
  std::vector<double> prior_center, prior_weight;
  if (opt->use_motion_priors)
    for (const auto& kv : sd->views) {
      const r3d_sfm_data::View& v = kv.second;
      if (!(v.priors && v.use_pose_center)) continue;
      auto pit = F.pose_index.find(v.id_pose);
      if (pit == F.pose_index.end() || !F.intr_index.count(v.id_intrinsic)) continue;  // IsPoseAndIntrinsicDefined
      prior_cam.push_back(pit->second);
      prior_center.insert(prior_center.end(), v.pose_center, v.pose_center + 3);
      prior_weight.insert(prior_weight.end(), v.center_weight, v.center_weight + 3);
    }
  r3d_ba_problem p;
  std::memset(&p, 0, sizeof(p));
  p.n_cams = (uint32_t)F.pose_index.size();
  p.n_pts = (uint32_t)F.lm_ids.size();
  p.n_intr = (uint32_t)F.intr_index.size();
  p.n_obs = F.obs_cam.size();
  p.poses = F.poses.data(); p.intrinsics = F.intr.data(); p.points = F.X.data();
  p.obs_cam = F.obs_cam.data(); p.obs_pt = obs_pt.data(); p.cam_intr = F.cam_intr.data(); p.obs_xy = F.obs_xy.data();
  p.intr_model = F.model.data();
  p.intrinsics_ext = F.ext.data();
  p.n_priors = (uint32_t)prior_cam.size();
  p.prior_cam = prior_cam.data(); p.prior_center = prior_center.data(); p.prior_weight = prior_weight.data();
  const int rc = r3d_bundle_adjust(ctx, &p, &opt->solver, summary, nullptr);
  if (rc) return rc;
  // ---- write back (Adjust updates the camera poses, intrinsics and structure with the refined values) ----------------
  const double* ps = F.poses.data();
  for (auto& kv : sd->poses) {
    r3d_sfm::angle_axis_to_rotation(ps, kv.second.R);
    r3d_sfm::center_of(kv.second.R, ps + 3, kv.second.C);
    ps += 6;
  }
  if (opt->solver.refine_intrinsics) {
    const double* q = F.intr.data();
    for (auto& kv : sd->intrinsics) {
      kv.second.focal = q[0]; kv.second.ppx = q[1]; kv.second.ppy = q[2];
      for (size_t k = 0; k < kv.second.disto.size() && k < 3; ++k) kv.second.disto[k] = q[3 + k];
      q += 6;
    }
  }
  const double* X = F.X.data();
  for (auto& kv : sd->structure) {
    std::memcpy(kv.second.X, X, 3 * sizeof(double));
    X += 3;
  }
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; } catch (...) { return R3D_ERR_INVALID; }
