// r3d_sfm.h -- openMVG::sfm::SfM_Data as the library holds it, and its flat form for the device code (sfm_scene.cpp).
#pragma once
#include <cmath>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "../../include/r3dgpu.h"

struct r3d_sfm_data {
  std::string root_path;
  struct View {
    std::string local_path, filename;
    uint32_t width = 0, height = 0, id_view = 0, id_intrinsic = 0, id_pose = 0;
    bool priors = false;            // openMVG::sfm::ViewPriors (GPS pose-centre prior)
    bool use_pose_center = false;
    double center_weight[3] = {1.0, 1.0, 1.0}, pose_center[3] = {0.0, 0.0, 0.0};
  };
  struct Intrinsic {
    int model = R3D_CAM_PINHOLE_RADIAL3;
    uint32_t width = 0, height = 0;
    double focal = 0, ppx = 0, ppy = 0;
    std::vector<double> disto;      // K1: 1, K3: 3, Brown T2: 5 (k1 k2 k3 t1 t2), fisheye: 4
  };
  struct Pose { double R[9], C[3]; };
  struct Obs { uint32_t id_feat; double x[2]; };
  struct Landmark { double X[3]; std::map<uint32_t, Obs> obs; };
  std::map<uint32_t, View> views;
  std::map<uint32_t, Intrinsic> intrinsics;
  std::map<uint32_t, Pose> poses;
  std::map<uint32_t, Landmark> structure, control_points;
};


namespace r3d_sfm {

inline void angle_axis_to_rotation(const double* aa, double* R) {  // Rodrigues, row-major
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  double A, B;
  if (th2 > 1e-16) {
    const double th = std::sqrt(th2);
    A = std::sin(th) / th;
    B = (1.0 - std::cos(th)) / th2;
  } else {
    A = 1.0 - th2 / 6.0;
    B = 0.5 - th2 / 24.0;
  }
  const double x = aa[0], y = aa[1], z = aa[2];
  const double K[9] = {0, -z, y, z, 0, -x, -y, x, 0};
  const double K2[9] = {x * x - th2, x * y, x * z, x * y, y * y - th2, y * z, x * z, y * z, z * z - th2};
  for (int i = 0; i < 9; ++i) R[i] = ((i == 0 || i == 4 || i == 8) ? 1.0 : 0.0) + A * K[i] + B * K2[i];
}

// the centre C = -R^T t of the camera [R | t], R row-major
inline void center_of(const double* R, const double* t, double* C) {
  for (int i = 0; i < 3; ++i) C[i] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
}

// an intrinsic as the C ABI returns it, disto padded with zeros to 5
inline void to_c_intrinsic(uint32_t id, const r3d_sfm_data::Intrinsic& in, r3d_sfm_intrinsic* out) {
  out->id = id; out->model = in.model; out->width = in.width; out->height = in.height;
  out->focal = in.focal; out->ppx = in.ppx; out->ppy = in.ppy;
  for (int i = 0; i < 5; ++i) out->disto[i] = i < (int)in.disto.size() ? in.disto[i] : 0.0;
}

// The scene as bundle adjustment, triangulation and the outlier filters read it, with OpenMVG's BA parameterisation
// (SURVEY.md A.7): poses and intrinsics in id order, one landmark per structure entry, its observations in view order.
struct Flat {
  std::map<uint32_t, uint32_t> pose_index, intr_index;  // id -> index
  std::vector<double> poses;                            // 6 per pose: angle-axis(R) | t = -R C
  std::vector<double> intr, ext;                        // 6 | 2 per intrinsic: f ppx ppy disto[0..2] | disto[3..4]
  std::vector<uint8_t> model;                           // R3D_CAM_* per intrinsic
  std::vector<uint32_t> cam_intr;                       // intrinsic index per pose (0 for a pose nobody observes)
  std::vector<uint32_t> lm_ids;                         // landmark id per index
  std::vector<double> X;                                // 3 per landmark
  std::vector<uint64_t> obs_ofs;                        // observations of landmark l: [obs_ofs[l], obs_ofs[l + 1])
  std::vector<uint32_t> obs_cam, obs_view;              // pose index, view id per observation
  std::vector<double> obs_xy;                           // 2 per observation
};

// sd -> F (empty).  An observation of an unknown view, or of a view whose pose or intrinsic is undefined, is left out
// when skip_undefined (IsPoseAndIntrinsicDefined) and is R3D_ERR_INVALID otherwise.  The solvers keep one intrinsic
// group per pose (id_pose = id_view in every sfm_data the reference writes): a pose observed through two intrinsics
// is R3D_ERR_UNSUPPORTED.  The first of these defects in (landmark, view) order decides the code.
int flatten(const r3d_sfm_data& sd, bool skip_undefined, Flat& F);

}  // namespace r3d_sfm

