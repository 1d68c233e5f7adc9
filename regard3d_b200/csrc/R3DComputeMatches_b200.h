// R3DComputeMatches_b200.h -- C++ shim with the method set of the reference's R3DComputeMatches
// (src/R3DComputeMatches.h:30-74), implemented over the C ABI of libr3dgpu (include/r3dgpu.h).
//
// In the Regard3D tree this header replaces src/R3DComputeMatches.h: the caller
// (R3DComputeMatchesThread::Entry, src/threads/R3DComputeMatchesThread.cpp:91-108) compiles unchanged
// when the four Regard3D/OpenMVG types below are mapped with the typedef block at the bottom of
// INTEGRATION.md.  Here (no wxWidgets / OpenMVG in the build image) the same class is instantiated on
// plain std types so that it compiles and is exercised by tests.
#pragma once
#include <functional>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/r3dgpu.h"

namespace r3d_shim {

// Regard3DFeatures::R3DFParams (src/Regard3DFeatures.h:52-69), same field names
struct R3DFParams {
  std::vector<std::string> keypointDetectorList_;
  float threshold_ = 0.001f;
  int nFeatures_ = 20000;
  float distRatio_ = 0.6f;
  bool computeHomographyMatrix_ = true;
  bool computeFundalmentalMatrix_ = true;  // (sic) spelling of the reference
  bool computeEssentialMatrix_ = true;
};

// the R3DProjectPaths fields computeMatches() reads (src/R3DProject.h:39-65; used at
// src/R3DComputeMatches.cpp:1672-1673, :1748, :1780, :2121)
struct R3DProjectPaths {
  std::string relativeImagePath_;
  std::string relativeMatchesPath_;
  std::string matchesSfmDataFilename_;
  std::string matchesFFilename_;
  std::string matchesEFilename_;
  std::string matchesHFilename_;
  int pictureSetId_ = 0;
};

// ImageInfo fields the stage needs (src/utils/ImageInfo.h:23-40)
struct ImageInfo {
  std::string filename_;  // image%06d.jpg inside relativeImagePath_ (src/R3DProject.cpp:1042)
  int imageWidth_ = 0, imageHeight_ = 0;
  double focalLength_ = 0.0, sensorWidth_ = 0.0;  // mm, from EXIF + camera database; 0 = unknown (ImageInfo, src/R3DProject.h)
};
typedef std::vector<ImageInfo> ImageInfoVector;

typedef std::map<std::pair<uint32_t, uint32_t>, std::vector<r3d_indmatch>> PairWiseMatches;

class R3DComputeMatches {
 public:
  R3DComputeMatches();
  virtual ~R3DComputeMatches();

  // the reference passes its wx main frame and reports through sendUpdateProgressBarEvent
  // (src/Regard3DMainFrame.cpp:276-290); here any callable takes its place
  void setMainFrame(std::function<void(float, const std::string&)> progressSink);
  void addImages(const ImageInfoVector& iiv);

  // same signature and error convention (bool, true = OK) as src/R3DComputeMatches.h:50-51.
  // cameraModel is consumed by writeSfmData in the reference and not needed by the matching stages.
  bool computeMatches(R3DFParams& params, bool svgOutput, const R3DProjectPaths& paths, int cameraModel,
                      int matchingAlgorithm);

  // twin of R3DFeaturesThread::extractFeaturesAndDescriptors (src/threads/R3DFeaturesThread.cpp:128-209) for the
  // "Fast-AKAZE" detector list: images[v] is imageInfoVector_[v] decoded by the caller to float gray in [0, 1]
  // (width x height row-major, :161-191).  Writes <basename>.feat / .desc under paths.relativeMatchesPath_, fills
  // statistics_.numberOfKeypoints_ (image order) and reports 0.2 .. 0.6 through the progress sink.  Any other detector
  // list: false with lastError() set.
  bool extractFeatures(const std::vector<const float*>& images, const R3DFParams& params, const R3DProjectPaths& paths);

  void updateProgress(float progress, const std::string& msg);

  struct R3DComputeMatchesStatistics {
    std::vector<int> numberOfKeypoints_;
    PairWiseMatches putativeMatches_;
    PairWiseMatches fundamentalMatches_;
    PairWiseMatches essentialMatches_;
    PairWiseMatches homographyMatches_;
  };
  const R3DComputeMatchesStatistics& getStatistics() { return statistics_; }
  const std::string& lastError() const { return lastError_; }

 private:
  ImageInfoVector imageInfoVector_;
  std::function<void(float, const std::string&)> progressSink_;
  R3DComputeMatchesStatistics statistics_;
  std::string lastError_;
  r3d_ctx* ctx_ = nullptr;
};

}  // namespace r3d_shim
