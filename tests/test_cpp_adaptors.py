"""The header-only openMVG::matching::ArrayMatcher adaptor (regard3d_b200/csrc/ArrayMatcher_b200.h) compiles against a
stand-in of the two OpenMVG types it is instantiated with, links with libr3dgpu.so, and -- on a machine without a
H100 -- fails loudly (Build returns false, the error text says there is no CPU fallback)."""
import os
import subprocess
import textwrap

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

SRC = textwrap.dedent(r'''
    #include <cstdio>
    #include <vector>
    #include "regard3d_b200/csrc/ArrayMatcher_b200.h"
    // stand-ins with the shape of openMVG/matching/matching_interface.hpp, metric.hpp, indMatch.hpp
    namespace openMVG { namespace matching {
    struct IndMatch { IndMatch(uint32_t i = 0, uint32_t j = 0) : i_(i), j_(j) {} uint32_t i_, j_; };
    using IndMatches = std::vector<IndMatch>;
    template <typename T> struct L2 { typedef T ElementType; typedef float ResultType; };
    template <typename Scalar, typename Metric> class ArrayMatcher {
     public:
      using ScalarT = Scalar; using DistanceType = typename Metric::ResultType;
      virtual ~ArrayMatcher() = default;
      virtual bool Build(const Scalar* dataset, int nbRows, int dimension) = 0;
      virtual bool SearchNeighbour(const Scalar* query, int* indice, DistanceType* distance) = 0;
      virtual bool SearchNeighbours(const Scalar* query, int nbQuery, IndMatches* indices,
                                    std::vector<DistanceType>* distances, size_t NN) = 0;
    };
    }}
    using namespace openMVG::matching;
    using GpuMatcher = r3d_shim::ArrayMatcher_b200<float, L2<float>, ArrayMatcher<float, L2<float>>, IndMatch>;
    int main() {
      GpuMatcher m;
      ArrayMatcher<float, L2<float>>* base = &m;   // usable through the OpenMVG interface
      std::vector<float> db(8 * 4, 0.5f), q(2 * 4, 0.25f);
      const bool built = base->Build(db.data(), 8, 4);
      IndMatches idx; std::vector<float> dist;
      const bool ok = built && base->SearchNeighbours(q.data(), 2, &idx, &dist, 2);
      std::printf("built=%d searched=%d n=%zu err=%s\n", (int)built, (int)ok, idx.size(), m.lastError().c_str());
      return 0;
    }
''')


def _build_and_run(tmp_path):
    src = tmp_path / "adaptor.cpp"
    src.write_text(SRC)
    exe = tmp_path / "adaptor"
    libdir = os.path.join(ROOT, "regard3d_b200")
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lr3dgpu",
           "-Wl,-rpath," + libdir]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


def test_array_matcher_adaptor_compiles_links_and_fails_loudly_without_gpu(r3dlib, tmp_path):
    out = _build_and_run(tmp_path)
    import torch
    if torch.cuda.is_available():
        assert "built=1 searched=1 n=4" in out
    else:
        assert "built=0 searched=0" in out and "no CPU fallback" in out


@pytest.mark.gpu
def test_array_matcher_adaptor_runs_on_the_gpu(r3dlib, tmp_path):
    """The adaptor's GPU branch (Build -> r3d_upload_regions, SearchNeighbours -> r3d_search_neighbours) on hardware."""
    assert "built=1 searched=1 n=4" in _build_and_run(tmp_path)


BA_SRC = textwrap.dedent(r'''
    #include <cmath>
    #include <cstdio>
    #include <map>
    #include <memory>
    #include <vector>
    #include "regard3d_b200/csrc/Bundle_Adjustment_b200.h"
    // stand-ins with the shape of openMVG's sfm_data.hpp / sfm_view.hpp / Camera_Pinhole_Radial.hpp / pose3.hpp /
    // sfm_landmark.hpp / sfm_data_BA.hpp (only what the adaptor touches)
    namespace openMVG {
    using IndexT = uint32_t;
    struct Vec3 { double v[3]; double& operator[](int i) { return v[i]; } double operator[](int i) const { return v[i]; } };
    struct Vec2 { double v[2]; double operator[](int i) const { return v[i]; } };
    namespace cameras {
    enum EINTRINSIC { PINHOLE_CAMERA = 1, PINHOLE_CAMERA_RADIAL1, PINHOLE_CAMERA_RADIAL3, PINHOLE_CAMERA_BROWN, PINHOLE_CAMERA_FISHEYE };
    enum class Intrinsic_Parameter_Type : int { NONE = 1, ADJUST_FOCAL_LENGTH = 2, ADJUST_PRINCIPAL_POINT = 4, ADJUST_DISTORTION = 8, ADJUST_ALL = 14 };
    struct IntrinsicBase {
      unsigned w_ = 0, h_ = 0; std::vector<double> params;   // f, ppx, ppy, k...
      virtual ~IntrinsicBase() = default;
      virtual EINTRINSIC getType() const = 0;
      std::vector<double> getParams() const { return params; }
      bool updateFromParams(const std::vector<double>& p) { params = p; return true; }
    };
    struct Pinhole_Intrinsic_Radial_K3 : IntrinsicBase { EINTRINSIC getType() const override { return PINHOLE_CAMERA_RADIAL3; } };
    }
    namespace geometry { struct Pose3 { double R[9]; double C[3]; const double* rotation() const { return R; } const double* center() const { return C; } }; }
    namespace sfm {
    struct View { IndexT id_view, id_intrinsic, id_pose, ui_width, ui_height; virtual ~View() = default; };
    struct ViewPriors : View { bool b_use_pose_center_ = false; Vec3 center_weight_{{1, 1, 1}}, pose_center_{{0, 0, 0}}; };
    struct Observation { Vec2 x; IndexT id_feat; };
    struct Landmark { Vec3 X; std::map<IndexT, Observation> obs; };
    struct SfM_Data {
      std::map<IndexT, std::shared_ptr<View>> views;
      std::map<IndexT, std::shared_ptr<cameras::IntrinsicBase>> intrinsics;
      std::map<IndexT, geometry::Pose3> poses;
      std::map<IndexT, Landmark> structure;
    };
    struct Optimize_Options { cameras::Intrinsic_Parameter_Type intrinsics_opt = cameras::Intrinsic_Parameter_Type::ADJUST_ALL; bool use_motion_priors_opt = false; };
    }}
    using namespace openMVG;
    // accessor shims: the only OpenMVG-specific code a maintainer writes
    struct Traits {
      static void view(const sfm::View& v, r3d_sfm_view* o) {
        o->id_view = v.id_view; o->id_intrinsic = v.id_intrinsic; o->id_pose = v.id_pose; o->width = v.ui_width; o->height = v.ui_height;
        const auto* p = dynamic_cast<const sfm::ViewPriors*>(&v);
        o->has_prior = (p && p->b_use_pose_center_) ? 1 : 0;
        for (int i = 0; i < 3; ++i) { o->center_weight[i] = p ? p->center_weight_[i] : 1.0; o->pose_center[i] = p ? p->pose_center_[i] : 0.0; }
      }
      static bool intrinsic(const cameras::IntrinsicBase& c, r3d_sfm_intrinsic* o) {
        const std::vector<double> p = c.getParams();
        o->model = (int)c.getType(); o->width = c.w_; o->height = c.h_; o->focal = p[0]; o->ppx = p[1]; o->ppy = p[2];
        for (size_t k = 3; k < p.size() && k < 8; ++k) o->disto[k - 3] = p[k];
        return o->model >= 1 && o->model <= 5;
      }
      static void set_intrinsic(cameras::IntrinsicBase& c, const r3d_sfm_intrinsic& in) {
        std::vector<double> p = c.getParams();
        p[0] = in.focal; p[1] = in.ppx; p[2] = in.ppy;
        for (size_t k = 3; k < p.size() && k < 8; ++k) p[k] = in.disto[k - 3];
        c.updateFromParams(p);
      }
      static void pose(const geometry::Pose3& p, double* R, double* C) { for (int i = 0; i < 9; ++i) R[i] = p.rotation()[i]; for (int i = 0; i < 3; ++i) C[i] = p.center()[i]; }
      static void set_pose(geometry::Pose3& p, const double* R, const double* C) { for (int i = 0; i < 9; ++i) p.R[i] = R[i]; for (int i = 0; i < 3; ++i) p.C[i] = C[i]; }
      static bool refine_intrinsics(const sfm::Optimize_Options& o) { return o.intrinsics_opt != cameras::Intrinsic_Parameter_Type::NONE; }
      static bool use_motion_priors(const sfm::Optimize_Options& o) { return o.use_motion_priors_opt; }
    };
    using GpuBA = r3d_shim::Bundle_Adjustment_b200<sfm::SfM_Data, sfm::Optimize_Options, Traits>;

    static double rms(const sfm::SfM_Data& s) {   // pinhole reprojection (k = 0 in this scene)
      double acc = 0; size_t n = 0;
      for (const auto& kv : s.structure) for (const auto& ob : kv.second.obs) {
        const auto& ps = s.poses.at(s.views.at(ob.first)->id_pose); const auto p = s.intrinsics.at(0)->getParams();
        double d[3] = {kv.second.X[0] - ps.C[0], kv.second.X[1] - ps.C[1], kv.second.X[2] - ps.C[2]}, c[3];
        for (int i = 0; i < 3; ++i) c[i] = ps.R[3 * i] * d[0] + ps.R[3 * i + 1] * d[1] + ps.R[3 * i + 2] * d[2];
        const double u = p[1] + p[0] * c[0] / c[2] - ob.second.x[0], v = p[2] + p[0] * c[1] / c[2] - ob.second.x[1];
        acc += u * u + v * v; ++n;
      }
      return std::sqrt(acc / n);
    }
    int main() {
      sfm::SfM_Data s;
      auto cam = std::make_shared<cameras::Pinhole_Intrinsic_Radial_K3>();
      cam->w_ = 1000; cam->h_ = 800; cam->params = {1010.0, 500.0, 400.0, 0.0, 0.0, 0.0};   // true focal 1000
      s.intrinsics[0] = cam;
      for (IndexT v = 0; v < 4; ++v) {
        auto vw = std::make_shared<sfm::ViewPriors>();
        vw->id_view = vw->id_pose = v; vw->id_intrinsic = 0; vw->ui_width = 1000; vw->ui_height = 800;
        s.views[v] = vw;
        geometry::Pose3 p{}; p.R[0] = p.R[4] = p.R[8] = 1.0; p.C[0] = 0.5 * v + (v ? 0.01 : 0.0); p.C[1] = 0.02 * v; p.C[2] = 0.0;
        s.poses[v] = p;
      }
      unsigned seed = 12345; auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) / 16777216.0; };
      for (IndexT k = 0; k < 60; ++k) {
        sfm::Landmark lm; const double X[3] = {rnd() * 4 - 1, rnd() * 2 - 1, 5 + 3 * rnd()};
        for (IndexT v = 0; v < 4; ++v) {                                         // exact projections from the TRUE cameras
          const double cx = 0.5 * v, cy = 0.02 * v;
          sfm::Observation ob; ob.id_feat = k; ob.x = {{500 + 1000 * (X[0] - cx) / X[2], 400 + 1000 * (X[1] - cy) / X[2]}};
          lm.obs[v] = ob;
        }
        lm.X = {{X[0] + 0.02 * (rnd() - 0.5), X[1] + 0.02 * (rnd() - 0.5), X[2] + 0.05 * (rnd() - 0.5)}};
        s.structure[k] = lm;
      }
      const double before = rms(s);
      GpuBA ba;
      const bool ok = ba.Adjust(s, sfm::Optimize_Options());
      std::printf("ok=%d before=%.4f after=%.6f iters=%u err=%s\n", (int)ok, before, ok ? rms(s) : -1.0, ba.summary().iterations,
                  ba.lastError().c_str());
      return 0;
    }
''')


def _build_ba(tmp_path):
    src = tmp_path / "ba_adaptor.cpp"
    src.write_text(BA_SRC)
    exe = tmp_path / "ba_adaptor"
    libdir = os.path.join(ROOT, "regard3d_b200")
    p = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-I", ROOT, str(src), "-o", str(exe), "-L", libdir, "-lr3dgpu",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


def test_bundle_adjustment_adaptor_compiles_links_and_fails_loudly_without_gpu(r3dlib, tmp_path):
    """Bundle_Adjustment_b200 (flatten / unflatten of an SfM_Data stand-in) compiles against OpenMVG-shaped types."""
    out = _build_ba(tmp_path)
    import torch
    if not torch.cuda.is_available():
        assert "ok=0" in out and "no CPU fallback" in out


@pytest.mark.gpu
def test_bundle_adjustment_adaptor_refines_a_scene_on_the_gpu(r3dlib, tmp_path):
    out = _build_ba(tmp_path)
    assert "ok=1" in out, out
    before = float(out.split("before=")[1].split()[0])
    after = float(out.split("after=")[1].split()[0])
    assert before > 1.0 and after < 1e-3 * before, out                 # noise-free observations: BA returns to ~0
