// features_io.cpp -- KeypointSet::saveToBinFile (src/threads/R3DFeaturesThread.cpp:200): openMVG's saveFeatsToFile
// (SIOPointFeature's operator<<: "x y scale orientation\n") and saveDescsToBinFile (a size_t count, then the raw
// float32 rows), byte for byte.
#include "r3d_internal.cuh"

#include <fstream>
#include <locale>

namespace r3d {

const char* save_features(const char* feat_path, const char* desc_path, const float* xyso, const float* desc, uint64_t n,
                          uint32_t dim) {
  {
    std::ofstream f(feat_path);
    if (!f.is_open()) return feat_path;
    f.imbue(std::locale::classic());  // a global locale with a decimal comma would change the text
    for (uint64_t i = 0; i < n; ++i)
      f << xyso[4 * i] << " " << xyso[4 * i + 1] << " " << xyso[4 * i + 2] << " " << xyso[4 * i + 3] << "\n";
    f.close();
    if (!f) return feat_path;
  }
  std::ofstream d(desc_path, std::ios::out | std::ios::binary);
  if (!d.is_open()) return desc_path;
  const std::size_t card = (std::size_t)n;
  d.write((const char*)&card, sizeof(card));
  if (n) d.write((const char*)desc, (std::streamsize)(n * dim * sizeof(float)));
  d.close();
  return d ? nullptr : desc_path;
}

}  // namespace r3d

extern "C" int r3d_save_features(const char* feat_path, const char* desc_path, const float* xyso, const float* desc,
                                 uint64_t n, uint32_t dim) {
  if (!feat_path || !desc_path || (n && (!xyso || !desc)) || dim == 0)
    return r3d::fail(nullptr, R3D_ERR_INVALID, "r3d_save_features: bad arguments");
  if (const char* bad = r3d::save_features(feat_path, desc_path, xyso, desc, n, dim))
    return r3d::fail(nullptr, R3D_ERR_IO, std::string("r3d_save_features: cannot write ") + bad);
  return R3D_OK;
}
