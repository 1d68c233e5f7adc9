// oracle_export.cpp -- CPU ORACLE (test infrastructure; see oracle.h) of what follows the SfM engine:
//   orc_colorize_plan          OpenMVGHelper::ColorizeTracks (src/utils/OpenMVGHelper.cpp:2453-2560) with its own
//                              containers: the remaining tracks in a std::set, the per-view counts in a std::map, the
//                              most represented view by std::partial_sort of one (count, index) packet under
//                              `a.val > b.val` (OpenMVG's sort_index_helper with nbuplet = 1)
//   orc_write_colorized_ply    plyHelper::exportToPly with colours (SfMPlyHelper.hpp:62-116) through std::ofstream
//   orc_undistort_image        OpenMVG 1.4 UndistortImage with black fill, as DESIGN.md 2.4 reads it
// Compile with -ffp-contract=off (export.mk).
#include "oracle_detmath.hpp"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <fstream>
#include <iomanip>
#include <limits>
#include <map>
#include <set>
#include <vector>

namespace {

struct Packet {  // stl::indexed_sort::sort_index_packet_descend<IndexT, IndexT>
  uint32_t val, index;
};
bool operator<(const Packet& a, const Packet& b) { return a.val > b.val; }

}  // namespace

extern "C" {

// views: n_views ids with their sizes; landmarks: n_lm ids, observations of landmark l in [obs_ofs[l], obs_ofs[l + 1])
// as (view id, x, y).  Outputs as r3d_sfm_colorize_plan.  -1: an unknown view, a landmark without observations or an
// observation whose truncated position lies outside its view.
int orc_colorize_plan(uint32_t n_views, const uint32_t* view_ids, const uint32_t* widths, const uint32_t* heights,
                      uint32_t n_lm, const uint32_t* lm_ids, const uint64_t* obs_ofs, const uint32_t* obs_view,
                      const double* obs_xy, uint32_t* round_view, uint32_t* n_rounds, uint32_t* lm_round, int32_t* lm_pixel) {
  std::map<uint32_t, std::pair<uint32_t, uint32_t>> views;
  for (uint32_t v = 0; v < n_views; ++v) views[view_ids[v]] = {widths[v], heights[v]};
  std::map<uint32_t, std::map<uint32_t, std::pair<double, double>>> landmarks;
  for (uint32_t l = 0; l < n_lm; ++l) {
    auto& obs = landmarks[lm_ids[l]];
    for (uint64_t o = obs_ofs[l]; o < obs_ofs[l + 1]; ++o) {
      const auto it = views.find(obs_view[o]);
      if (it == views.end()) return -1;
      const double x = obs_xy[2 * o], y = obs_xy[2 * o + 1];
      if (!(x > -1.0 && x < (double)it->second.first && y > -1.0 && y < (double)it->second.second)) return -1;
      obs[obs_view[o]] = {x, y};
    }
    if (obs.empty()) return -1;
  }
  std::map<uint32_t, uint32_t> contiguous;
  uint32_t cpt = 0;
  for (const auto& kv : landmarks) contiguous[kv.first] = cpt++;
  std::set<uint32_t> remaining;
  for (const auto& kv : landmarks) remaining.insert(kv.first);
  uint32_t round = 0;
  while (!remaining.empty()) {
    std::map<uint32_t, uint32_t> cardinal;
    for (uint32_t t : remaining)
      for (const auto& ob : landmarks.at(t)) {
        if (cardinal.find(ob.first) == cardinal.end()) cardinal[ob.first] = 1;
        else ++cardinal[ob.first];
      }
    std::vector<uint32_t> vec_cardinal;
    for (const auto& kv : cardinal) vec_cardinal.push_back(kv.second);
    std::vector<Packet> packets(vec_cardinal.size());
    for (size_t i = 0; i < packets.size(); ++i) packets[i] = {vec_cardinal[i], (uint32_t)i};
    std::partial_sort(packets.begin(), packets.begin() + 1, packets.end());
    auto itv = cardinal.begin();
    std::advance(itv, packets[0].index);
    const uint32_t view = itv->first;
    round_view[round] = view;
    std::set<uint32_t> to_remove;
    for (uint32_t t : remaining) {
      const auto& obs = landmarks.at(t);
      const auto it = obs.find(view);
      if (it != obs.end()) {
        const uint32_t c = contiguous[t];
        lm_round[c] = round;
        lm_pixel[2 * c] = (int32_t)it->second.first;   // image(pt.y(), pt.x()): the index conversion truncates
        lm_pixel[2 * c + 1] = (int32_t)it->second.second;
        to_remove.insert(t);
      }
    }
    for (uint32_t t : to_remove) remaining.erase(t);
    ++round;
  }
  *n_rounds = round;
  return 0;
}

// X: n_lm x 3; colors: n_lm x 3 or NULL; centers: n_poses x 3.  -1: the file could not be written.
int orc_write_colorized_ply(uint32_t n_lm, const double* X, const uint8_t* colors, uint32_t n_poses, const double* centers,
                            const char* path) {
  std::ofstream out(path);
  if (!out.is_open()) return -1;
  out << "ply" << '\n' << "format ascii 1.0" << '\n' << "element vertex " << (size_t)n_lm + n_poses << '\n'
      << "property double x" << '\n' << "property double y" << '\n' << "property double z" << '\n'
      << "property uchar red" << '\n' << "property uchar green" << '\n' << "property uchar blue" << '\n' << "end_header"
      << std::endl;
  out << std::fixed << std::setprecision(std::numeric_limits<double>::digits10 + 1);
  for (uint32_t i = 0; i < n_lm; ++i) {
    out << X[3 * i] << ' ' << X[3 * i + 1] << ' ' << X[3 * i + 2] << ' ';
    if (colors)
      out << (int)colors[3 * i] << ' ' << (int)colors[3 * i + 1] << ' ' << (int)colors[3 * i + 2] << "\n";
    else
      out << "255 255 255\n";
  }
  for (uint32_t i = 0; i < n_poses; ++i)
    out << centers[3 * i] << ' ' << centers[3 * i + 1] << ' ' << centers[3 * i + 2] << ' ' << "0 255 0\n";
  out.flush();
  const bool ok = out.good();
  out.close();
  return ok ? 0 : -1;
}

// model 1..5 (EINTRINSIC), disto as r3d_sfm_intrinsic; rgb / out: h x w x 3.  -1: unknown model.
int orc_undistort_image(int model, double f, double ppx, double ppy, const double* disto, const uint8_t* rgb, uint32_t w,
                        uint32_t h, uint8_t* out) {
  if (model < 1 || model > 5) return -1;
  const size_t bytes = (size_t)w * h * 3;
  if (model == 1) {  // have_disto() false: image_ud = imageIn
    std::copy(rgb, rgb + bytes, out);
    return 0;
  }
  std::fill(out, out + bytes, (uint8_t)0);
  const int W = (int)w, H = (int)h;
  for (int j = 0; j < H; ++j) {
    for (int i = 0; i < W; ++i) {
      // ima2cam
      const double px = ((double)i - ppx) / f, py = ((double)j - ppy) / f;
      double qx, qy;  // add_disto
      if (model == 2) {
        const double k1 = disto[0];
        const double r2 = px * px + py * py;
        const double r_coeff = (1. + k1 * r2);
        qx = px * r_coeff;
        qy = py * r_coeff;
      } else if (model == 3) {
        const double k1 = disto[0], k2 = disto[1], k3 = disto[2];
        const double r2 = px * px + py * py, r4 = r2 * r2, r6 = r4 * r2;
        const double r_coeff = (1. + k1 * r2 + k2 * r4 + k3 * r6);
        qx = px * r_coeff;
        qy = py * r_coeff;
      } else if (model == 4) {
        const double k1 = disto[0], k2 = disto[1], k3 = disto[2], t1 = disto[3], t2 = disto[4];
        const double r2 = px * px + py * py, r4 = r2 * r2, r6 = r4 * r2;
        const double k_diff = (k1 * r2 + k2 * r4 + k3 * r6);
        const double t_x = t2 * (r2 + 2 * px * px) + 2 * t1 * px * py;
        const double t_y = t1 * (r2 + 2 * py * py) + 2 * t2 * px * py;
        qx = px + (px * k_diff + t_x);
        qy = py + (py * k_diff + t_y);
      } else {
        const double eps = 1e-8;
        const double k1 = disto[0], k2 = disto[1], k3 = disto[2], k4 = disto[3];
        const double r = std::sqrt(px * px + py * py);
        const double theta = orc::det::atan_pos(r);
        const double theta2 = theta * theta, theta3 = theta2 * theta, theta4 = theta2 * theta2, theta5 = theta4 * theta,
                     theta7 = theta3 * theta3 * theta, theta8 = theta4 * theta4, theta9 = theta8 * theta;
        const double theta_dist = theta + k1 * theta3 + k2 * theta5 + k3 * theta7 + k4 * theta9;
        const double inv_r = r > eps ? 1.0 / r : 1.0;
        const double cdist = r > eps ? theta_dist * inv_r : 1.0;
        qx = px * cdist;
        qy = py * cdist;
      }
      // cam2ima
      const double dx = f * qx + ppx, dy = f * qy + ppy;
      // Contains((int)dy, (int)dx), without converting a double the int cannot hold
      if (!(dx > -1.0 && dx < (double)W && dy > -1.0 && dy < (double)H)) continue;
      // Sampler2d<SamplerLinear>(in, (float)dy, (float)dx)
      const float y = (float)dy, x = (float)dx;
      const float coefs_x[2] = {1.0f - (x - std::floor(x)), x - std::floor(x)};
      const float coefs_y[2] = {1.0f - (y - std::floor(y)), y - std::floor(y)};
      const int grid_x = (int)std::floor(x), grid_y = (int)std::floor(y);
      double res[3] = {0.0, 0.0, 0.0}, total_weight = 0.0;
      for (int a = 0; a < 2; ++a) {
        const int cur_i = grid_y + a;
        if (cur_i < 0 || cur_i >= H) continue;
        for (int b = 0; b < 2; ++b) {
          const int cur_j = grid_x + b;
          if (cur_j < 0 || cur_j >= W) continue;
          const float wgt = coefs_x[b] * coefs_y[a];
          const uint8_t* p = rgb + 3 * ((size_t)cur_i * w + (size_t)cur_j);
          for (int c = 0; c < 3; ++c) res[c] += (double)p[c] * (double)wgt;
          total_weight += (double)wgt;
        }
      }
      if (total_weight <= 0.2) continue;  // T(): black
      if (total_weight != 1.0)
        for (double& v : res) v /= total_weight;
      uint8_t* o = out + 3 * ((size_t)j * w + (size_t)i);
      for (int c = 0; c < 3; ++c) o[c] = (uint8_t)std::min(std::max(res[c], 0.0), 255.0);
    }
  }
  return 0;
}

}  // extern "C"
