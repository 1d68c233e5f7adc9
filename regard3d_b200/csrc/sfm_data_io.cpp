// sfm_data_io.cpp -- the reference's native on-disk containers, without OpenMVG / cereal (SURVEY.md 8f-2, App. B.4):
//   sfm_data.bin   openMVG::sfm::Save / Load(SfM_Data, "*.bin", flags)  -- written by R3DProject::writeSfmData
//                  (src/R3DProject.cpp:1118-1306, Save at :1298-1302 with VIEWS | INTRINSICS), read back by
//                  R3DComputeMatches (src/R3DComputeMatches.cpp:1755) and the triangulation thread
//                  (src/threads/R3DTriangulationThread.cpp:403), written with ALL after SfM (:453-455)
//   matches.*.bin  openMVG::matching::Save / Load(PairWiseMatches, "*.bin")
// Both are cereal PortableBinary archives.  cereal and OpenMVG are un-vendored dependencies (not in /root/reference,
// not in this image), so the byte layout below restates their published serialisation code:
//   cereal 1.x  archives/portable_binary.hpp   1 byte "archive is little endian", then raw little-endian scalars
//               types/string.hpp, vector.hpp   uint64 size tag, then the elements (arithmetic vectors: raw block)
//               types/map.hpp, utility.hpp     uint64 size tag, then key, value per item; pair: first, second
//               types/memory.hpp + polymorphic.hpp   shared_ptr<T>: uint32 polymorphic_id (0x40000000 = "static type",
//               else a per-archive type id, MSB set on first use and followed by the registered name), then uint32
//               pointer id (MSB set on first use, then the object)
//   OpenMVG 1.4 sfm/sfm_data_io_cereal.hpp (version string "0.3", root_path, views, intrinsics, extrinsics,
//               structure, control_points), sfm_view.hpp / sfm_view_priors.hpp, cameras/Camera_Pinhole*.hpp
//               (registered names "pinhole", "pinhole_radial_k1", "pinhole_radial_k3", "pinhole_brown_t2",
//               "pinhole_fisheye"), geometry/pose3.hpp, sfm_landmark.hpp, matching/indMatch.hpp
// PARITY UNPINNED: no reference-produced file exists in /root/reference and none can be produced here; the tests pin
// the writer against a byte stream assembled independently from this specification (tests/test_sfm_data_io.py).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/r3dgpu.h"
#include "r3d_matches.h"
#include "r3d_sfm.h"

namespace {

const uint32_t kMsb = 0x80000000u, kMsb2 = 0x40000000u;

struct Writer {
  std::vector<unsigned char> b;
  void raw(const void* p, size_t n) { const unsigned char* c = (const unsigned char*)p; b.insert(b.end(), c, c + n); }
  void u8(uint8_t v) { b.push_back(v); }
  void u32(uint32_t v) { raw(&v, 4); }
  void u64(uint64_t v) { raw(&v, 8); }
  void f64(double v) { raw(&v, 8); }
  void str(const std::string& s) { u64(s.size()); raw(s.data(), s.size()); }
  void vec(const double* v, size_t n) { u64(n); raw(v, 8 * n); }
};

struct Reader {
  const unsigned char* p;
  const unsigned char* end;
  bool ok = true;
  bool need(size_t n) { if ((size_t)(end - p) < n) { ok = false; return false; } return true; }
  void raw(void* d, size_t n) { if (need(n)) { std::memcpy(d, p, n); p += n; } else std::memset(d, 0, n); }
  uint8_t u8() { uint8_t v = 0; raw(&v, 1); return v; }
  uint32_t u32() { uint32_t v = 0; raw(&v, 4); return v; }
  uint64_t u64() { uint64_t v = 0; raw(&v, 8); return v; }
  double f64() { double v = 0; raw(&v, 8); return v; }
  std::string str() {
    const uint64_t n = u64();
    if (!need(n)) return std::string();
    std::string s((const char*)p, (size_t)n);
    p += n;
    return s;
  }
  bool vec(double* d, size_t n_expected) {  // a std::vector<double> of a known length
    const uint64_t n = u64();
    if (n != n_expected) { ok = false; return false; }
    raw(d, 8 * n_expected);
    return ok;
  }
  std::vector<double> vec_any(size_t max_n) {
    const uint64_t n = u64();
    std::vector<double> v;
    if (n > max_n || !need(8 * n)) { ok = false; return v; }
    v.resize(n);
    raw(v.data(), 8 * n);
    return v;
  }
};

const char* model_name(int model) {
  switch (model) {
    case R3D_CAM_PINHOLE: return "pinhole";
    case R3D_CAM_PINHOLE_RADIAL1: return "pinhole_radial_k1";
    case R3D_CAM_PINHOLE_RADIAL3: return "pinhole_radial_k3";
    case R3D_CAM_PINHOLE_BROWN: return "pinhole_brown_t2";
    case R3D_CAM_PINHOLE_FISHEYE: return "pinhole_fisheye";
  }
  return nullptr;
}
int model_of_name(const std::string& n) {
  for (int m = R3D_CAM_PINHOLE; m <= R3D_CAM_PINHOLE_FISHEYE; ++m)
    if (n == model_name(m)) return m;
  return 0;
}
size_t disto_count(int model) {
  switch (model) {
    case R3D_CAM_PINHOLE_RADIAL1: return 1;
    case R3D_CAM_PINHOLE_RADIAL3: return 3;
    case R3D_CAM_PINHOLE_BROWN: return 5;
    case R3D_CAM_PINHOLE_FISHEYE: return 4;
  }
  return 0;
}

// per-archive bookkeeping of cereal's OutputArchive: polymorphic names and shared pointers get running ids from 1
struct SaveIds {
  std::map<std::string, uint32_t> names;
  uint32_t next_name = 1, next_ptr = 1;
  void polymorphic(Writer& w, const char* name) {
    auto it = names.find(name);
    if (it != names.end()) { w.u32(it->second); return; }
    const uint32_t id = next_name++;
    names[name] = id;
    w.u32(id | kMsb);
    w.str(name);
  }
  void pointer(Writer& w) { w.u32((next_ptr++) | kMsb); }  // every object of these containers is saved once
};

void write_landmarks(Writer& w, const std::map<uint32_t, r3d_sfm_data::Landmark>& L) {
  w.u64(L.size());
  for (const auto& kv : L) {
    w.u32(kv.first);
    w.vec(kv.second.X, 3);
    w.u64(kv.second.obs.size());
    for (const auto& ob : kv.second.obs) {
      w.u32(ob.first);
      w.u32(ob.second.id_feat);
      w.vec(ob.second.x, 2);
    }
  }
}

bool read_landmarks(Reader& r, std::map<uint32_t, r3d_sfm_data::Landmark>& L) {
  const uint64_t n = r.u64();
  for (uint64_t k = 0; k < n && r.ok; ++k) {
    const uint32_t id = r.u32();
    r3d_sfm_data::Landmark lm;
    r.vec(lm.X, 3);
    const uint64_t no = r.u64();
    for (uint64_t q = 0; q < no && r.ok; ++q) {
      const uint32_t view = r.u32();
      r3d_sfm_data::Obs ob;
      ob.id_feat = r.u32();
      r.vec(ob.x, 2);
      lm.obs[view] = ob;
    }
    L[id] = std::move(lm);
  }
  return r.ok;
}

int serialize(const r3d_sfm_data& sd, uint32_t parts, std::vector<unsigned char>& out) {
  Writer w;
  SaveIds ids;
  w.u8(1);  // PortableBinaryOutputArchive: "this archive is little endian"
  w.str("0.3");
  w.str(sd.root_path);
  // views: Hash_Map<IndexT, std::shared_ptr<View>>
  if (parts & R3D_SFM_VIEWS) {
    w.u64(sd.views.size());
    for (const auto& kv : sd.views) {
      const r3d_sfm_data::View& v = kv.second;
      w.u32(kv.first);
      // ViewPriors::save writes its prior only when it is in use, and a binary reader cannot tell: a prior that is
      // switched off is stored as a plain View
      const bool as_priors = v.priors && v.use_pose_center;
      if (as_priors) ids.polymorphic(w, "view_priors");
      else w.u32(kMsb2);  // the pointee IS an openMVG::sfm::View: no polymorphic cast needed
      ids.pointer(w);
      w.str(v.local_path); w.str(v.filename);
      w.u32(v.width); w.u32(v.height); w.u32(v.id_view); w.u32(v.id_intrinsic); w.u32(v.id_pose);
      if (as_priors) {
        w.u8(1);
        w.vec(v.center_weight, 3);
        w.vec(v.pose_center, 3);
      }
    }
  } else {
    w.u64(0);
  }
  // intrinsics: Hash_Map<IndexT, std::shared_ptr<IntrinsicBase>> (abstract base: always through the name binding)
  if (parts & R3D_SFM_INTRINSICS) {
    w.u64(sd.intrinsics.size());
    for (const auto& kv : sd.intrinsics) {
      const r3d_sfm_data::Intrinsic& in = kv.second;
      const char* name = model_name(in.model);
      if (!name || in.disto.size() != disto_count(in.model)) return R3D_ERR_INVALID;
      w.u32(kv.first);
      ids.polymorphic(w, name);
      ids.pointer(w);
      w.u32(in.width); w.u32(in.height);
      w.f64(in.focal);
      const double pp[2] = {in.ppx, in.ppy};
      w.vec(pp, 2);
      if (!in.disto.empty()) w.vec(in.disto.data(), in.disto.size());
    }
  } else {
    w.u64(0);
  }
  // extrinsics: Hash_Map<IndexT, geometry::Pose3>: rotation as 3 row vectors, then the centre
  if (parts & R3D_SFM_EXTRINSICS) {
    w.u64(sd.poses.size());
    for (const auto& kv : sd.poses) {
      w.u32(kv.first);
      w.u64(3);
      for (int r = 0; r < 3; ++r) w.vec(kv.second.R + 3 * r, 3);
      w.vec(kv.second.C, 3);
    }
  } else {
    w.u64(0);
  }
  if (parts & R3D_SFM_STRUCTURE) write_landmarks(w, sd.structure); else w.u64(0);
  if (parts & R3D_SFM_CONTROL_POINTS) write_landmarks(w, sd.control_points); else w.u64(0);
  out.swap(w.b);
  return R3D_OK;
}

int deserialize(const unsigned char* data, size_t size, r3d_sfm_data& sd) {
  Reader r{data, data + size};
  if (r.u8() != 1) return R3D_ERR_UNSUPPORTED;  // a big-endian writer
  const std::string version = r.str();
  if (!r.ok || (version != "0.3" && version != "0.2")) return R3D_ERR_UNSUPPORTED;
  sd.root_path = r.str();
  std::map<uint32_t, std::string> names;  // InputArchive: polymorphic id -> name
  auto read_poly = [&](std::string& name, bool& static_type) {
    const uint32_t id = r.u32();
    static_type = (id & kMsb2) != 0;
    name.clear();
    if (static_type) return;
    if (id & kMsb) { name = r.str(); names[id & ~kMsb] = name; }
    else { auto it = names.find(id); if (it == names.end()) r.ok = false; else name = it->second; }
  };
  // views
  uint64_t n = r.u64();
  for (uint64_t k = 0; k < n && r.ok; ++k) {
    const uint32_t key = r.u32();
    std::string name;
    bool st = false;
    read_poly(name, st);
    if (!st && name != "view_priors" && name != "view") { r.ok = false; break; }
    const uint32_t pid = r.u32();
    if (!(pid & kMsb)) { r.ok = false; break; }  // a view shared by two map entries never occurs
    r3d_sfm_data::View v;
    v.local_path = r.str(); v.filename = r.str();
    v.width = r.u32(); v.height = r.u32(); v.id_view = r.u32(); v.id_intrinsic = r.u32(); v.id_pose = r.u32();
    if (name == "view_priors") {
      v.priors = true;
      v.use_pose_center = r.u8() != 0;
      if (v.use_pose_center) { r.vec(v.center_weight, 3); r.vec(v.pose_center, 3); }
    }
    sd.views[key] = std::move(v);
  }
  // intrinsics
  n = r.u64();
  for (uint64_t k = 0; k < n && r.ok; ++k) {
    const uint32_t key = r.u32();
    std::string name;
    bool st = false;
    read_poly(name, st);
    const int model = model_of_name(name);
    if (st || !model) { r.ok = false; break; }
    const uint32_t pid = r.u32();
    if (!(pid & kMsb)) { r.ok = false; break; }
    r3d_sfm_data::Intrinsic in;
    in.model = model;
    in.width = r.u32(); in.height = r.u32();
    in.focal = r.f64();
    double pp[2];
    r.vec(pp, 2);
    in.ppx = pp[0]; in.ppy = pp[1];
    if (disto_count(model)) {
      in.disto = r.vec_any(16);
      if (in.disto.size() != disto_count(model)) r.ok = false;
    }
    sd.intrinsics[key] = std::move(in);
  }
  // extrinsics
  n = r.u64();
  for (uint64_t k = 0; k < n && r.ok; ++k) {
    const uint32_t key = r.u32();
    r3d_sfm_data::Pose ps;
    if (r.u64() != 3) { r.ok = false; break; }
    for (int row = 0; row < 3; ++row) r.vec(ps.R + 3 * row, 3);
    r.vec(ps.C, 3);
    sd.poses[key] = ps;
  }
  if (r.ok) read_landmarks(r, sd.structure);
  if (r.ok && version != "0.1") read_landmarks(r, sd.control_points);
  return r.ok ? R3D_OK : R3D_ERR_IO;
}

bool read_file(const char* path, std::vector<unsigned char>& buf) {
  std::ifstream f(path, std::ios::binary);
  if (!f.is_open()) return false;
  f.seekg(0, std::ios::end);
  const std::streamoff n = f.tellg();
  f.seekg(0, std::ios::beg);
  if (n < 0) return false;
  buf.resize((size_t)n);
  if (n) f.read((char*)buf.data(), n);
  return (bool)f;
}

bool ends_with(const char* s, const char* suf) {
  const size_t a = std::strlen(s), b = std::strlen(suf);
  return a >= b && std::strcmp(s + a - b, suf) == 0;
}

}  // namespace

extern "C" {

int r3d_sfm_data_create(r3d_sfm_data** out) try {
  if (!out) return R3D_ERR_INVALID;
  *out = new r3d_sfm_data();
  return R3D_OK;
} catch (...) { return R3D_ERR_NOMEM; }

void r3d_sfm_data_free(r3d_sfm_data* sd) { delete sd; }

int r3d_sfm_data_load(const char* path, r3d_sfm_data** out) try {
  if (!path || !out) return R3D_ERR_INVALID;
  *out = nullptr;
  std::vector<unsigned char> buf;
  if (!read_file(path, buf)) return R3D_ERR_IO;
  std::unique_ptr<r3d_sfm_data> sd(new r3d_sfm_data());
  const int rc = deserialize(buf.data(), buf.size(), *sd);
  if (rc) return rc;
  *out = sd.release();
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; } catch (...) { return R3D_ERR_IO; }

int r3d_sfm_data_save(const r3d_sfm_data* sd, const char* path, uint32_t parts) try {
  if (!sd || !path) return R3D_ERR_INVALID;
  std::vector<unsigned char> buf;
  const int rc = serialize(*sd, parts, buf);
  if (rc) return rc;
  std::ofstream f(path, std::ios::binary);
  if (!f.is_open()) return R3D_ERR_IO;
  f.write((const char*)buf.data(), (std::streamsize)buf.size());
  return f.good() ? R3D_OK : R3D_ERR_IO;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; } catch (...) { return R3D_ERR_IO; }

const char* r3d_sfm_root_path(const r3d_sfm_data* sd) { return sd ? sd->root_path.c_str() : ""; }
int r3d_sfm_set_root_path(r3d_sfm_data* sd, const char* p) try {
  if (!sd || !p) return R3D_ERR_INVALID;
  sd->root_path = p;
  return R3D_OK;
} catch (...) { return R3D_ERR_NOMEM; }

uint32_t r3d_sfm_num_views(const r3d_sfm_data* sd) { return sd ? (uint32_t)sd->views.size() : 0; }
uint32_t r3d_sfm_num_intrinsics(const r3d_sfm_data* sd) { return sd ? (uint32_t)sd->intrinsics.size() : 0; }
uint32_t r3d_sfm_num_poses(const r3d_sfm_data* sd) { return sd ? (uint32_t)sd->poses.size() : 0; }
uint32_t r3d_sfm_num_landmarks(const r3d_sfm_data* sd, int control_points) {
  return sd ? (uint32_t)(control_points ? sd->control_points.size() : sd->structure.size()) : 0;
}

int r3d_sfm_add_view(r3d_sfm_data* sd, const r3d_sfm_view* v) try {
  if (!sd || !v) return R3D_ERR_INVALID;
  r3d_sfm_data::View w;
  w.local_path = v->local_path ? v->local_path : "";
  w.filename = v->filename ? v->filename : "";
  w.width = v->width; w.height = v->height; w.id_view = v->id_view; w.id_intrinsic = v->id_intrinsic; w.id_pose = v->id_pose;
  w.priors = v->has_prior != 0;
  w.use_pose_center = v->has_prior != 0;
  for (int i = 0; i < 3; ++i) { w.center_weight[i] = v->center_weight[i]; w.pose_center[i] = v->pose_center[i]; }
  sd->views[v->id_view] = std::move(w);
  return R3D_OK;
} catch (...) { return R3D_ERR_NOMEM; }

int r3d_sfm_get_view(const r3d_sfm_data* sd, uint32_t k, r3d_sfm_view* out) {
  if (!sd || !out || k >= sd->views.size()) return R3D_ERR_INVALID;
  auto it = sd->views.begin();
  std::advance(it, k);
  const r3d_sfm_data::View& w = it->second;
  out->local_path = w.local_path.c_str(); out->filename = w.filename.c_str();
  out->width = w.width; out->height = w.height; out->id_view = w.id_view; out->id_intrinsic = w.id_intrinsic; out->id_pose = w.id_pose;
  out->has_prior = (w.priors && w.use_pose_center) ? 1 : 0;
  for (int i = 0; i < 3; ++i) { out->center_weight[i] = w.center_weight[i]; out->pose_center[i] = w.pose_center[i]; }
  return R3D_OK;
}

int r3d_sfm_add_intrinsic(r3d_sfm_data* sd, const r3d_sfm_intrinsic* in) try {
  if (!sd || !in || !model_name(in->model)) return R3D_ERR_INVALID;
  r3d_sfm_data::Intrinsic w;
  w.model = in->model; w.width = in->width; w.height = in->height; w.focal = in->focal; w.ppx = in->ppx; w.ppy = in->ppy;
  w.disto.assign(in->disto, in->disto + disto_count(in->model));
  sd->intrinsics[in->id] = std::move(w);
  return R3D_OK;
} catch (...) { return R3D_ERR_NOMEM; }

int r3d_sfm_get_intrinsic(const r3d_sfm_data* sd, uint32_t k, r3d_sfm_intrinsic* out) {
  if (!sd || !out || k >= sd->intrinsics.size()) return R3D_ERR_INVALID;
  auto it = sd->intrinsics.begin();
  std::advance(it, k);
  r3d_sfm::to_c_intrinsic(it->first, it->second, out);
  return R3D_OK;
}

int r3d_sfm_add_pose(r3d_sfm_data* sd, const r3d_sfm_pose* p) try {
  if (!sd || !p) return R3D_ERR_INVALID;
  r3d_sfm_data::Pose w;
  std::memcpy(w.R, p->rotation, sizeof(w.R));
  std::memcpy(w.C, p->center, sizeof(w.C));
  sd->poses[p->id] = w;
  return R3D_OK;
} catch (...) { return R3D_ERR_NOMEM; }

int r3d_sfm_get_pose(const r3d_sfm_data* sd, uint32_t k, r3d_sfm_pose* out) {
  if (!sd || !out || k >= sd->poses.size()) return R3D_ERR_INVALID;
  auto it = sd->poses.begin();
  std::advance(it, k);
  out->id = it->first;
  std::memcpy(out->rotation, it->second.R, sizeof(out->rotation));
  std::memcpy(out->center, it->second.C, sizeof(out->center));
  return R3D_OK;
}

int r3d_sfm_add_landmark(r3d_sfm_data* sd, int control_point, uint32_t id, const double X[3], const r3d_sfm_observation* obs,
                         uint32_t n_obs) try {
  if (!sd || !X || (n_obs && !obs)) return R3D_ERR_INVALID;
  r3d_sfm_data::Landmark lm;
  std::memcpy(lm.X, X, sizeof(lm.X));
  for (uint32_t k = 0; k < n_obs; ++k) {
    r3d_sfm_data::Obs ob;
    ob.id_feat = obs[k].id_feat; ob.x[0] = obs[k].x[0]; ob.x[1] = obs[k].x[1];
    lm.obs[obs[k].id_view] = ob;
  }
  (control_point ? sd->control_points : sd->structure)[id] = std::move(lm);
  return R3D_OK;
} catch (...) { return R3D_ERR_NOMEM; }

int r3d_sfm_get_landmark(const r3d_sfm_data* sd, int control_point, uint32_t k, uint32_t* id, double X[3],
                         r3d_sfm_observation* obs, uint32_t obs_cap, uint32_t* n_obs) {
  if (!sd) return R3D_ERR_INVALID;
  const auto& L = control_point ? sd->control_points : sd->structure;
  if (k >= L.size()) return R3D_ERR_INVALID;
  auto it = L.begin();
  std::advance(it, k);
  if (id) *id = it->first;
  if (X) std::memcpy(X, it->second.X, 3 * sizeof(double));
  if (n_obs) *n_obs = (uint32_t)it->second.obs.size();
  if (obs) {
    uint32_t q = 0;
    for (const auto& ob : it->second.obs) {
      if (q >= obs_cap) break;
      obs[q].id_view = ob.first; obs[q].id_feat = ob.second.id_feat; obs[q].x[0] = ob.second.x[0]; obs[q].x[1] = ob.second.x[1];
      ++q;
    }
  }
  return R3D_OK;
}

// ---- matches.*.bin: cereal PortableBinary of std::map<std::pair<IndexT, IndexT>, std::vector<IndMatch>> -------------
int r3d_save_matches_bin(const r3d_matches* m, const char* path) try {
  if (!m || !path) return R3D_ERR_INVALID;
  Writer w;
  const uint64_t P = m->pairs.size() / 2;
  w.u8(1);
  w.u64(P);
  for (uint64_t k = 0; k < P; ++k) {
    w.u32(m->pairs[2 * k]); w.u32(m->pairs[2 * k + 1]);
    w.u64(m->per[k].size());
    w.raw(m->per[k].data(), m->per[k].size() * sizeof(r3d_indmatch));  // IndMatch::serialize: i_, j_ (uint32 each)
  }
  std::ofstream f(path, std::ios::binary);
  if (!f.is_open()) return R3D_ERR_IO;
  f.write((const char*)w.b.data(), (std::streamsize)w.b.size());
  return f.good() ? R3D_OK : R3D_ERR_IO;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; } catch (...) { return R3D_ERR_IO; }

int r3d_load_matches_bin(const char* path, r3d_matches** out) try {
  if (!path || !out) return R3D_ERR_INVALID;
  *out = nullptr;
  std::vector<unsigned char> buf;
  if (!read_file(path, buf)) return R3D_ERR_IO;
  Reader r{buf.data(), buf.data() + buf.size()};
  if (r.u8() != 1) return R3D_ERR_UNSUPPORTED;
  const uint64_t P = r.u64();
  std::map<std::pair<uint32_t, uint32_t>, std::vector<r3d_indmatch>> mp;
  for (uint64_t k = 0; k < P && r.ok; ++k) {
    const uint32_t I = r.u32(), J = r.u32();
    const uint64_t n = r.u64();
    if (!r.need(n * sizeof(r3d_indmatch))) break;
    std::vector<r3d_indmatch> v((size_t)n);
    r.raw(v.data(), n * sizeof(r3d_indmatch));
    mp[{I, J}] = std::move(v);
  }
  if (!r.ok) return R3D_ERR_IO;
  std::unique_ptr<r3d_matches> m(new r3d_matches());
  for (auto& kv : mp) m->push(kv.first.first, kv.first.second, std::move(kv.second));
  *out = m.release();
  return R3D_OK;
} catch (const std::bad_alloc&) { return R3D_ERR_NOMEM; } catch (...) { return R3D_ERR_IO; }

// matching::Save / Load pick the format from the extension (".txt" / ".bin"), like the reference's calls do
int r3d_save_matches(const r3d_matches* m, const char* path) {
  if (!path) return R3D_ERR_INVALID;
  if (ends_with(path, ".bin")) return r3d_save_matches_bin(m, path);
  if (ends_with(path, ".txt")) return r3d_save_matches_txt(m, path);
  return R3D_ERR_UNSUPPORTED;
}
int r3d_load_matches(const char* path, r3d_matches** out) {
  if (!path) return R3D_ERR_INVALID;
  if (ends_with(path, ".bin")) return r3d_load_matches_bin(path, out);
  if (ends_with(path, ".txt")) return r3d_load_matches_txt(path, out);
  return R3D_ERR_UNSUPPORTED;
}

}  // extern "C"
