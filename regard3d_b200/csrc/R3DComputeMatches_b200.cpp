// R3DComputeMatches_b200.cpp -- see the header.  Mirrors R3DComputeMatches::computeMatches()
// (src/R3DComputeMatches.cpp:1667-2256) from "load regions" on; every numeric stage is a call into
// the C ABI (no OpenMVG, no CPU fallback: without a B200 the constructor's context creation fails
// and computeMatches() returns false).
#include "R3DComputeMatches_b200.h"

#include <algorithm>
#include <cstring>

namespace r3d_shim {

namespace {
void progress_trampoline(float f, const char* msg, void* user) {
  static_cast<R3DComputeMatches*>(user)->updateProgress(f, msg ? msg : "");
}
std::string strip_ext(const std::string& s) {
  const size_t p = s.find_last_of('.');
  return p == std::string::npos ? s : s.substr(0, p);
}
void to_map(const r3d_matches* m, PairWiseMatches& out) {
  out.clear();
  const uint64_t P = r3d_matches_num_pairs(m);
  for (uint64_t k = 0; k < P; ++k) {
    uint32_t I, J;
    const r3d_indmatch* p;
    uint64_t n;
    r3d_matches_get_pair(m, k, &I, &J, &p, &n);
    out[{I, J}] = std::vector<r3d_indmatch>(p, p + n);
  }
}
}  // namespace

R3DComputeMatches::R3DComputeMatches() {
  if (r3d_create(nullptr, 0, &ctx_) != R3D_OK) {
    ctx_ = nullptr;
    lastError_ = r3d_last_error(nullptr);
  }
}

R3DComputeMatches::~R3DComputeMatches() { r3d_destroy(ctx_); }

void R3DComputeMatches::setMainFrame(std::function<void(float, const std::string&)> progressSink) {
  progressSink_ = std::move(progressSink);
}

void R3DComputeMatches::addImages(const ImageInfoVector& iiv) { imageInfoVector_ = iiv; }

void R3DComputeMatches::updateProgress(float progress, const std::string& msg) {
  if (progressSink_) progressSink_(progress, msg);
}

bool R3DComputeMatches::computeMatches(R3DFParams& params, bool svgOutput, const R3DProjectPaths& paths,
                                       int /*cameraModel*/, int matchingAlgorithm) {
  if (!ctx_) return false;
  const uint32_t n = (uint32_t)imageInfoVector_.size();
  std::vector<std::string> bases(n);
  std::vector<const char*> base_ptrs(n);
  std::vector<r3d_view_info> views(n);
  for (uint32_t v = 0; v < n; ++v) {
    bases[v] = strip_ext(imageInfoVector_[v].filename_);  // <basename>.feat / .desc (R3DFeaturesThread.cpp:132-136)
    base_ptrs[v] = bases[v].c_str();
    views[v].width = (uint32_t)imageInfoVector_[v].imageWidth_;
    views[v].height = (uint32_t)imageInfoVector_[v].imageHeight_;
    // pinhole K of the view exactly as R3DProject::writeSfmData builds it (src/R3DProject.cpp:1143-1159)
    const ImageInfo& ii = imageInfoVector_[v];
    const int wmax = std::max(ii.imageWidth_, ii.imageHeight_);
    views[v].focal = (ii.focalLength_ > 0 && ii.sensorWidth_ > 0) ? wmax * ii.focalLength_ / ii.sensorWidth_ : wmax * 1.1;
    views[v].ppx = static_cast<double>(ii.imageWidth_) / 2.0;
    views[v].ppy = static_cast<double>(ii.imageHeight_) / 2.0;
  }
  r3d_cm_params p;
  p.dist_ratio = params.distRatio_;
  p.compute_fundamental = params.computeFundalmentalMatrix_ ? 1 : 0;
  p.compute_essential = params.computeEssentialMatrix_ ? 1 : 0;
  p.compute_homography = params.computeHomographyMatrix_ ? 1 : 0;
  p.matching_algorithm = matchingAlgorithm;
  p.descriptor_dim = 144;
  p.svg_output = svgOutput ? 1 : 0;
  r3d_cm_paths cp;
  cp.matches_dir = paths.relativeMatchesPath_.c_str();
  cp.image_basenames = base_ptrs.data();
  cp.views = views.data();
  cp.n_views = n;
  cp.matches_f_filename = paths.matchesFFilename_.empty() ? nullptr : paths.matchesFFilename_.c_str();
  cp.matches_h_filename = paths.matchesHFilename_.empty() ? nullptr : paths.matchesHFilename_.c_str();
  cp.matches_e_filename = paths.matchesEFilename_.empty() ? nullptr : paths.matchesEFilename_.c_str();
  std::vector<uint32_t> kp(n, 0);
  r3d_cm_stats st;
  std::memset(&st, 0, sizeof(st));
  st.n_views = n;
  st.number_of_keypoints = kp.data();
  const int rc = r3d_compute_matches(ctx_, &p, &cp, progress_trampoline, this, &st);
  if (rc != R3D_OK) {
    lastError_ = r3d_last_error(ctx_);
    return false;
  }
  statistics_.numberOfKeypoints_.assign(kp.begin(), kp.end());
  // the statistics maps are filled like the reference does (src/R3DComputeMatches.cpp:2079, :2128),
  // from the files just written
  r3d_matches* m = nullptr;
  if (r3d_load_matches_txt((paths.relativeMatchesPath_ + "/matches.putative.txt").c_str(), &m) == R3D_OK) {
    to_map(m, statistics_.putativeMatches_);
    r3d_free_matches(m);
  }
  if (params.computeFundalmentalMatrix_) {
    const std::string f = paths.matchesFFilename_.empty() ? paths.relativeMatchesPath_ + "/matches.f.txt" : paths.matchesFFilename_;
    if (r3d_load_matches_txt(f.c_str(), &m) == R3D_OK) {
      to_map(m, statistics_.fundamentalMatches_);
      r3d_free_matches(m);
    }
  }
  if (params.computeEssentialMatrix_) {
    const std::string f = paths.matchesEFilename_.empty() ? paths.relativeMatchesPath_ + "/matches.e.txt" : paths.matchesEFilename_;
    if (r3d_load_matches_txt(f.c_str(), &m) == R3D_OK) {
      to_map(m, statistics_.essentialMatches_);
      r3d_free_matches(m);
    }
  }
  if (params.computeHomographyMatrix_) {
    const std::string f = paths.matchesHFilename_.empty() ? paths.relativeMatchesPath_ + "/matches.h.txt" : paths.matchesHFilename_;
    if (r3d_load_matches_txt(f.c_str(), &m) == R3D_OK) {
      to_map(m, statistics_.homographyMatches_);
      r3d_free_matches(m);
    }
  }
  return true;
}

bool R3DComputeMatches::extractFeatures(const std::vector<const float*>& images, const R3DFParams& params,
                                        const R3DProjectPaths& paths) {
  if (!ctx_) return false;
  if (params.keypointDetectorList_ != std::vector<std::string>{"Fast-AKAZE"}) {
    lastError_ = "extractFeatures: only the detector list {\"Fast-AKAZE\"} runs on the GPU";
    return false;
  }
  const uint32_t n = (uint32_t)imageInfoVector_.size();
  if (images.size() != n) {
    lastError_ = "extractFeatures: one image per ImageInfo expected";
    return false;
  }
  std::vector<std::string> bases(n);
  std::vector<const char*> base_ptrs(n);
  std::vector<uint32_t> widths(n), heights(n);
  for (uint32_t v = 0; v < n; ++v) {
    bases[v] = strip_ext(imageInfoVector_[v].filename_);  // R3DFeaturesThread.cpp:132-136
    base_ptrs[v] = bases[v].c_str();
    widths[v] = (uint32_t)imageInfoVector_[v].imageWidth_;
    heights[v] = (uint32_t)imageInfoVector_[v].imageHeight_;
  }
  r3d_extract_options o;
  r3d_extract_default_options(&o);
  o.akaze.threshold = params.threshold_;
  o.out_dir = paths.relativeMatchesPath_.c_str();
  o.basenames = base_ptrs.data();
  r3d_features* f = nullptr;
  const int rc = r3d_extract_features(ctx_, images.data(), widths.data(), heights.data(), n, &o, progress_trampoline,
                                      this, &f);
  if (rc != R3D_OK) {
    lastError_ = r3d_last_error(ctx_);
    return false;
  }
  statistics_.numberOfKeypoints_.resize(n);
  for (uint32_t v = 0; v < n; ++v) statistics_.numberOfKeypoints_[v] = (int)r3d_features_count(f, v);
  r3d_free_features(f);
  return true;
}

}  // namespace r3d_shim

// C hook so the Python tests can drive the shim's feature extraction: detector "Fast-AKAZE" unless detector is given
extern "C" int r3d_shim_extract_features(const char* matches_dir, const char* const* image_filenames, const float* const* images,
                                         const uint32_t* widths, const uint32_t* heights, uint32_t n, float threshold,
                                         const char* detector, uint32_t* n_keypoints_out, float* last_progress) {
  r3d_shim::R3DComputeMatches cm;
  float last = -1.f;
  cm.setMainFrame([&](float f, const std::string&) { last = f; });
  r3d_shim::ImageInfoVector iiv(n);
  for (uint32_t v = 0; v < n; ++v) {
    iiv[v].filename_ = image_filenames[v];
    iiv[v].imageWidth_ = (int)widths[v];
    iiv[v].imageHeight_ = (int)heights[v];
  }
  cm.addImages(iiv);
  r3d_shim::R3DFParams params;
  params.keypointDetectorList_ = {detector ? detector : "Fast-AKAZE"};
  params.threshold_ = threshold;
  r3d_shim::R3DProjectPaths paths;
  paths.relativeMatchesPath_ = matches_dir;
  const bool ok = cm.extractFeatures(std::vector<const float*>(images, images + n), params, paths);
  *last_progress = last;
  if (!ok) return -1;
  const auto& st = cm.getStatistics();
  for (uint32_t v = 0; v < n; ++v) n_keypoints_out[v] = (uint32_t)st.numberOfKeypoints_[v];
  return 0;
}

// C hook so the Python tests can drive the C++ shim end to end.
extern "C" int r3d_shim_compute_matches(const char* matches_dir, const char* const* image_filenames, const uint32_t* widths,
                                        const uint32_t* heights, uint32_t n, float dist_ratio, int matching_algorithm,
                                        uint32_t* n_keypoints_out, uint64_t* putative_pairs, uint64_t* f_pairs,
                                        float* last_progress) {
  r3d_shim::R3DComputeMatches cm;
  float last = -1.f;
  cm.setMainFrame([&](float f, const std::string&) { last = f; });
  r3d_shim::ImageInfoVector iiv(n);
  for (uint32_t v = 0; v < n; ++v) {
    iiv[v].filename_ = image_filenames[v];
    iiv[v].imageWidth_ = (int)widths[v];
    iiv[v].imageHeight_ = (int)heights[v];
  }
  cm.addImages(iiv);
  r3d_shim::R3DFParams params;
  params.distRatio_ = dist_ratio;
  r3d_shim::R3DProjectPaths paths;
  paths.relativeMatchesPath_ = matches_dir;
  const bool ok = cm.computeMatches(params, false, paths, 3, matching_algorithm);
  if (!ok) return -1;
  const auto& st = cm.getStatistics();
  for (uint32_t v = 0; v < n && v < st.numberOfKeypoints_.size(); ++v) n_keypoints_out[v] = (uint32_t)st.numberOfKeypoints_[v];
  *putative_pairs = st.putativeMatches_.size();
  *f_pairs = st.fundamentalMatches_.size();
  *last_progress = last;
  return 0;
}
