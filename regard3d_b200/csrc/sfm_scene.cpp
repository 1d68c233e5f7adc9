// sfm_scene.cpp -- the SfM_Data scene flattened for the device code: r3d_sfm_bundle_adjust (sfm_ba.cpp),
// r3d_sfm_structure_from_tracks and r3d_sfm_remove_outliers (sfm_structure.cu) all read it through r3d_sfm::flatten.
#include "r3d_sfm.h"
#include "relpose_math.cuh"

namespace r3d_sfm {

int flatten(const r3d_sfm_data& sd, bool skip_undefined, Flat& F) {
  for (const auto& kv : sd.poses) {
    F.pose_index[kv.first] = (uint32_t)F.pose_index.size();
    double aa[3];
    r3d::rp::rotation_to_angle_axis(kv.second.R, aa);
    const double* R = kv.second.R;
    const double* C = kv.second.C;
    F.poses.insert(F.poses.end(), {aa[0], aa[1], aa[2], -(R[0] * C[0] + R[1] * C[1] + R[2] * C[2]),
                                   -(R[3] * C[0] + R[4] * C[1] + R[5] * C[2]), -(R[6] * C[0] + R[7] * C[1] + R[8] * C[2])});
  }
  for (const auto& kv : sd.intrinsics) {
    F.intr_index[kv.first] = (uint32_t)F.intr_index.size();
    const r3d_sfm_data::Intrinsic& in = kv.second;
    double p6[6] = {in.focal, in.ppx, in.ppy, 0, 0, 0}, e2[2] = {0, 0};
    for (size_t k = 0; k < in.disto.size(); ++k) {
      if (k < 3) p6[3 + k] = in.disto[k];
      else e2[k - 3] = in.disto[k];
    }
    F.intr.insert(F.intr.end(), p6, p6 + 6);
    F.ext.insert(F.ext.end(), e2, e2 + 2);
    F.model.push_back((uint8_t)in.model);
  }
  F.cam_intr.assign(F.pose_index.size(), 0u);
  std::vector<uint8_t> cam_set(F.pose_index.size(), 0);
  F.obs_ofs.push_back(0);
  for (const auto& kv : sd.structure) {
    F.lm_ids.push_back(kv.first);
    F.X.insert(F.X.end(), kv.second.X, kv.second.X + 3);
    for (const auto& ob : kv.second.obs) {
      const auto vit = sd.views.find(ob.first);
      const bool known = vit != sd.views.end();
      const auto pit = known ? F.pose_index.find(vit->second.id_pose) : F.pose_index.end();
      const auto iit = known ? F.intr_index.find(vit->second.id_intrinsic) : F.intr_index.end();
      if (pit == F.pose_index.end() || iit == F.intr_index.end()) {
        if (skip_undefined) continue;
        return R3D_ERR_INVALID;
      }
      if (cam_set[pit->second] && F.cam_intr[pit->second] != iit->second) return R3D_ERR_UNSUPPORTED;
      cam_set[pit->second] = 1;
      F.cam_intr[pit->second] = iit->second;
      F.obs_cam.push_back(pit->second);
      F.obs_view.push_back(ob.first);
      F.obs_xy.push_back(ob.second.x[0]);
      F.obs_xy.push_back(ob.second.x[1]);
    }
    F.obs_ofs.push_back(F.obs_cam.size());
  }
  return R3D_OK;
}

}  // namespace r3d_sfm
