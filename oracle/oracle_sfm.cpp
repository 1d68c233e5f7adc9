// oracle_sfm.cpp -- CPU ORACLE (test infrastructure; see oracle.h) of the steps either side of bundle adjustment that
// SURVEY.md 8f-3 names: track building, triangulation of the tracks from known poses, outlier rejection.
//
// Reference call sites: openMVG::tracks::TracksBuilder Build / Filter / ExportToSTL and
// TracksUtilsMap::GetTracksInImages are called by Regard3D itself (src/threads/PreviewGeneratorThread.cpp:345-358);
// triangulation and the outlier filters run inside the OpenMVG SfM engines the reference drives
// (src/threads/R3DTriangulationThread.cpp:418-441, :492-512).  All of it is un-vendored OpenMVG 1.4, restated from its
// published sources (tracks/tracks.hpp + union_find.hpp, multiview/triangulation_nview.hpp `Triangulation`,
// sfm/sfm_data_triangulation.cpp SfM_Data_Structure_Computation_Blind, sfm/sfm_data_filters.hpp).  PARITY UNPINNED.
#include "oracle.h"
#include "oracle_undistort.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <map>
#include <set>
#include <vector>

namespace orc {

// ---- union_find.hpp: union by rank + path compression --------------------------------------------------------------
struct UnionFind {
  std::vector<unsigned int> parent, rank, size;
  void InitSets(unsigned int n) {
    parent.resize(n); rank.assign(n, 0); size.assign(n, 1);
    for (unsigned int i = 0; i < n; ++i) parent[i] = i;
  }
  unsigned int Find(unsigned int i) {
    if (parent[i] != i) parent[i] = Find(parent[i]);
    return parent[i];
  }
  void Union(unsigned int i, unsigned int j) {
    i = Find(i); j = Find(j);
    if (i == j) return;
    if (rank[i] < rank[j]) { parent[i] = j; size[j] += size[i]; }
    else { parent[j] = i; size[i] += size[j]; if (rank[i] == rank[j]) ++rank[i]; }
  }
};

// TracksBuilder::Build + Filter(nLengthSupMin) + ExportToSTL: map track id -> map image id -> feature id.
// pairs / pair_ofs / m: a PairWiseMatches map in std::map order.
void tracks_build(const uint32_t* pairs, uint64_t P, const uint64_t* pair_ofs, const orc_indmatch* m, uint32_t min_length,
                  std::map<uint32_t, std::map<uint32_t, uint32_t>>& out) {
  typedef std::pair<uint32_t, uint32_t> Node;  // (image, feature)
  std::set<Node> all;
  for (uint64_t p = 0; p < P; ++p)
    for (uint64_t k = pair_ofs[p]; k < pair_ofs[p + 1]; ++k) {
      all.emplace(pairs[2 * p], m[k].i);
      all.emplace(pairs[2 * p + 1], m[k].j);
    }
  std::vector<Node> nodes(all.begin(), all.end());  // flat_pair_map: sorted, index = position
  auto index_of = [&](const Node& n) { return (unsigned int)(std::lower_bound(nodes.begin(), nodes.end(), n) - nodes.begin()); };
  UnionFind uf;
  uf.InitSets((unsigned int)nodes.size());
  for (uint64_t p = 0; p < P; ++p)
    for (uint64_t k = pair_ofs[p]; k < pair_ofs[p + 1]; ++k)
      uf.Union(index_of(Node(pairs[2 * p], m[k].i)), index_of(Node(pairs[2 * p + 1], m[k].j)));
  for (unsigned int k = 0; k < nodes.size(); ++k) uf.Find(k);  // every parent[] entry is now its root
  // Filter: tracks with an image id collision, and tracks that are too short
  std::map<unsigned int, std::set<unsigned int>> tracks;
  std::set<unsigned int> problematic;
  for (unsigned int k = 0; k < nodes.size(); ++k) {
    const unsigned int track_id = uf.parent[k];
    if (problematic.count(track_id)) continue;
    if (tracks[track_id].count(nodes[k].first)) problematic.insert(track_id);
    else tracks[track_id].insert(nodes[k].first);
  }
  for (const auto& val : tracks)
    if (val.second.size() < min_length) problematic.insert(val.first);
  const unsigned int kInvalid = std::numeric_limits<unsigned int>::max();
  for (unsigned int& root : uf.parent)
    if (root != kInvalid && problematic.count(root)) { uf.size[root] = 1; root = kInvalid; }
  out.clear();
  for (unsigned int k = 0; k < nodes.size(); ++k) {
    const unsigned int track_id = uf.parent[k];
    if (track_id != kInvalid && uf.size[track_id] > 1) out[track_id].insert(nodes[k]);
  }
}

// ---- geometry helpers -------------------------------------------------------------------------------------------------
namespace {
// radial K1 / K3 undistortion of a normalised point (Pinhole_Intrinsic_Radial_K*::remove_disto): bisection on the radius
double undistort_radius_factor(int model, const double* k, double r2d) {
  if (r2d == 0.0 || model < 2 || model > 3) return 1.0;
  auto disto = [&](double r2) {  // distoFunctor: r2 * c(r2)^2
    const double c = 1.0 + k[0] * r2 + (model == 3 ? k[1] * r2 * r2 + k[2] * r2 * r2 * r2 : 0.0);
    return r2 * c * c;
  };
  // bisection_Radius_Solve: bracket, then halve until |disto(r) - r2d| <= eps
  double lo = r2d, hi = r2d;
  while (disto(lo) > r2d) lo /= 1.05;
  while (disto(hi) < r2d) hi *= 1.05;
  const double eps = 1e-8;
  while (eps < hi - lo) {
    const double mid = .5 * (lo + hi);
    if (disto(mid) > r2d) hi = mid; else lo = mid;
  }
  return std::sqrt(.5 * (lo + hi) / r2d);
}
}  // namespace

// cam->get_ud_pixel(x): pixel without distortion.  Radial K1 / K3 by upstream's bisection; Brown T2 and fisheye by the
// resection oracle's Newton inverse (oracle_undistort.hpp).  intr: f ppx ppy k1 k2 k3; ext: t1 t2 (Brown) or k4 (fisheye)
void undistort_pixel(int model, const double* intr, const double* ext, const double* x, double* out) {
  const double f = intr[0], ppx = intr[1], ppy = intr[2];
  if (model == 4 || model == 5) {
    const double disto[5] = {intr[3], intr[4], intr[5], ext ? ext[0] : 0.0, ext ? ext[1] : 0.0};
    undistort_newton(model, f, ppx, ppy, disto, x[0], x[1], out, out + 1);
    return;
  }
  if (model < 2 || model > 3 || (intr[3] == 0.0 && intr[4] == 0.0 && intr[5] == 0.0)) { out[0] = x[0]; out[1] = x[1]; return; }
  const double xd = (x[0] - ppx) / f, yd = (x[1] - ppy) / f;
  const double s = undistort_radius_factor(model, intr + 3, xd * xd + yd * yd);
  out[0] = f * xd * s + ppx;
  out[1] = f * yd * s + ppy;
}

// multiview/triangulation_nview.hpp `Triangulation::compute(iter = 3)`: iteratively re-weighted inhomogeneous DLT.
// P: n projection matrices 3x4 (row-major), x: n x 2.  Returns X; *zmin = smallest depth.
void triangulate_nview(const double* P, const double* x, int n, double* X, double* zmin_out) {
  std::vector<double> w(n, 1.0);
  double zmin = 0;
  for (int it = 0; it < 3; ++it) {
    double AtA[9] = {0}, Atb[3] = {0};
    for (int i = 0; i < n; ++i) {
      const double* PM = P + 12 * i;
      const double px = x[2 * i], py = x[2 * i + 1], wi = w[i];
      double v1[3], v2[3];
      for (int j = 0; j < 3; ++j) {
        v1[j] = wi * (PM[j] - px * PM[8 + j]);
        v2[j] = wi * (PM[4 + j] - py * PM[8 + j]);
        Atb[j] += wi * (v1[j] * (px * PM[11] - PM[3]) + v2[j] * (py * PM[11] - PM[7]));
      }
      for (int k = 0; k < 3; ++k)
        for (int j = 0; j <= k; ++j) {
          const double v = v1[k] * v1[j] + v2[k] * v2[j];
          AtA[3 * k + j] += v;
          if (j < k) AtA[3 * j + k] += v;
        }
    }
    // X = AtA^-1 Atb (adjugate inverse of the symmetric 3x3)
    const double* a = AtA;
    const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
    const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
    const double inv[9] = {c00 / det, (a[2] * a[7] - a[1] * a[8]) / det, (a[1] * a[5] - a[2] * a[4]) / det,
                           c01 / det, (a[0] * a[8] - a[2] * a[6]) / det, (a[2] * a[3] - a[0] * a[5]) / det,
                           c02 / det, (a[1] * a[6] - a[0] * a[7]) / det, (a[0] * a[4] - a[1] * a[3]) / det};
    for (int i = 0; i < 3; ++i) X[i] = inv[3 * i] * Atb[0] + inv[3 * i + 1] * Atb[1] + inv[3 * i + 2] * Atb[2];
    zmin = std::numeric_limits<double>::max();
    for (int i = 0; i < n; ++i) {
      const double* PM = P + 12 * i;
      const double z = PM[8] * X[0] + PM[9] * X[1] + PM[10] * X[2] + PM[11];
      if (z < zmin) zmin = z;
      w[i] = 1.0 / z;
    }
  }
  *zmin_out = zmin;
}

}  // namespace orc

// ------------------------------------------------------------------------------------------------
extern "C" {

// CSR export of the track map: track_ofs[T+1], then (view, feat) pairs in map order; returns T (or -1 if cap too small)
int64_t orc_tracks_build(const uint32_t* pairs, uint64_t P, const uint64_t* pair_ofs, const orc_indmatch* m, uint32_t min_length,
                         uint32_t* track_ids, uint64_t* track_ofs, uint32_t* views, uint32_t* feats, uint64_t cap_tracks,
                         uint64_t cap_nodes) {
  std::map<uint32_t, std::map<uint32_t, uint32_t>> t;
  orc::tracks_build(pairs, P, pair_ofs, m, min_length, t);
  if (t.size() > cap_tracks) return -1;
  uint64_t k = 0, o = 0;
  for (const auto& kv : t) {
    if (o + kv.second.size() > cap_nodes) return -1;
    track_ids[k] = kv.first;
    track_ofs[k] = o;
    for (const auto& vf : kv.second) { views[o] = vf.first; feats[o] = vf.second; ++o; }
    ++k;
  }
  track_ofs[k] = o;
  return (int64_t)k;
}

// SfM_Data_Structure_Computation_Blind::triangulate on flat arrays: landmark l has observations obs_ofs[l]..obs_ofs[l+1]
// (camera index, pixel); cameras: pose (angle-axis | t) and intrinsic group (model, intr[6], ext[2] = t1 t2 | k4 0, or
// null for zeros).  ok[l] = 1 and X[l] set when >= 2 observations and the smallest depth is positive.
void orc_triangulate_landmarks(uint32_t n_lm, const uint64_t* obs_ofs, const uint32_t* obs_cam, const double* obs_xy,
                               const double* poses, const uint32_t* cam_intr, const double* intrinsics, const uint8_t* intr_model,
                               const double* intrinsics_ext, double* X, uint8_t* ok);
}

namespace {
void rodrigues(const double* aa, double* R) {
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  double A, B;
  if (th2 > 1e-16) { const double th = std::sqrt(th2); A = std::sin(th) / th; B = (1.0 - std::cos(th)) / th2; }
  else { A = 1.0 - th2 / 6.0; B = 0.5 - th2 / 24.0; }
  const double x = aa[0], y = aa[1], z = aa[2];
  const double K[9] = {0, -z, y, z, 0, -x, -y, x, 0};
  const double K2[9] = {x * x - th2, x * y, x * z, x * y, y * y - th2, y * z, x * z, y * z, z * z - th2};
  for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.0 : 0.0) + A * K[i] + B * K2[i];
}
}  // namespace

extern "C" {

void orc_triangulate_landmarks(uint32_t n_lm, const uint64_t* obs_ofs, const uint32_t* obs_cam, const double* obs_xy,
                               const double* poses, const uint32_t* cam_intr, const double* intrinsics, const uint8_t* intr_model,
                               const double* intrinsics_ext, double* X, uint8_t* ok) {
#pragma omp parallel for schedule(dynamic, 256)
  for (int64_t l = 0; l < (int64_t)n_lm; ++l) {
    const int n = (int)(obs_ofs[l + 1] - obs_ofs[l]);
    ok[l] = 0;
    if (n < 2) continue;
    std::vector<double> P(12 * (size_t)n), x(2 * (size_t)n);
    for (int t = 0; t < n; ++t) {
      const uint64_t o = obs_ofs[l] + t;
      const uint32_t c = obs_cam[o], g = cam_intr[c];
      const double* in = intrinsics + 6 * (size_t)g;
      double R[9];
      rodrigues(poses + 6 * (size_t)c, R);
      const double* tr = poses + 6 * (size_t)c + 3;
      // get_projective_equivalent: K [R | t]
      const double Kf = in[0], kx = in[1], ky = in[2];
      double* PM = &P[12 * (size_t)t];
      for (int j = 0; j < 3; ++j) {
        PM[j] = Kf * R[j] + kx * R[6 + j];
        PM[4 + j] = Kf * R[3 + j] + ky * R[6 + j];
        PM[8 + j] = R[6 + j];
      }
      PM[3] = Kf * tr[0] + kx * tr[2];
      PM[7] = Kf * tr[1] + ky * tr[2];
      PM[11] = tr[2];
      orc::undistort_pixel(intr_model ? intr_model[g] : 3, in, intrinsics_ext ? intrinsics_ext + 2 * (size_t)g : nullptr, obs_xy + 2 * o,
                           &x[2 * (size_t)t]);
    }
    double zmin;
    orc::triangulate_nview(P.data(), x.data(), n, X + 3 * l, &zmin);
    ok[l] = zmin > 0 ? 1 : 0;
  }
}

// sfm_data_filters.hpp on the same flat layout.  keep_obs[o] = 0 for observations whose pixel residual norm exceeds thr
// (RemoveOutliers_PixelResidualError); max_angle[l] = largest angle (degrees) between two observation rays
// (RemoveOutliers_AngleError compares it with dMinAcceptedAngle).
void orc_landmark_checks(uint32_t n_lm, const uint64_t* obs_ofs, const uint32_t* obs_cam, const double* obs_xy, const double* poses,
                         const uint32_t* cam_intr, const double* intrinsics, const uint8_t* intr_model, const double* intrinsics_ext,
                         const double* X, double thr_px, uint8_t* keep_obs, double* max_angle) {
  orc_ba_problem p;
  std::memset(&p, 0, sizeof(p));
#pragma omp parallel for schedule(dynamic, 256)
  for (int64_t l = 0; l < (int64_t)n_lm; ++l) {
    const int n = (int)(obs_ofs[l + 1] - obs_ofs[l]);
    std::vector<double> rays(3 * (size_t)n);
    for (int t = 0; t < n; ++t) {
      const uint64_t o = obs_ofs[l] + t;
      const uint32_t c = obs_cam[o], g = cam_intr[c];
      double r[2], J[30];
      orc_ba_jacobian_model(intr_model ? intr_model[g] : 3, intrinsics + 6 * (size_t)g, intrinsics_ext ? intrinsics_ext + 2 * (size_t)g : nullptr,
                            poses + 6 * (size_t)c, X + 3 * l, obs_xy + 2 * o, r, J);
      keep_obs[o] = std::sqrt(r[0] * r[0] + r[1] * r[1]) > thr_px ? 0 : 1;
      // ray from the camera centre to X, in world coordinates: X - C, C = -R^T t
      double R[9];
      rodrigues(poses + 6 * (size_t)c, R);
      const double* tr = poses + 6 * (size_t)c + 3;
      for (int i = 0; i < 3; ++i) rays[3 * (size_t)t + i] = X[3 * l + i] + (R[i] * tr[0] + R[3 + i] * tr[1] + R[6 + i] * tr[2]);
    }
    double best = 0.0;
    for (int a = 0; a < n; ++a)
      for (int b = a + 1; b < n; ++b) {
        const double* u = &rays[3 * (size_t)a];
        const double* v = &rays[3 * (size_t)b];
        const double d = u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
        const double nu = std::sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), nv = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        double cs = d / (nu * nv);
        cs = cs > 1.0 ? 1.0 : (cs < -1.0 ? -1.0 : cs);
        best = std::max(best, std::acos(cs) * 180.0 / M_PI);
      }
    max_angle[l] = best;
  }
}

}  // extern "C"
