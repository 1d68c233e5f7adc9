// context.cu -- context life-cycle, region upload and tensor-core operand preparation.
#include "r3d_internal.cuh"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <thread>

namespace r3d {

int operand_col_align() {
  static int a = -1;
  if (a < 0) {
    const char* e = getenv("R3D_KP_ALIGN");
    a = (e && atoi(e) == 16) ? 16 : 64;
  }
  return a;
}

static std::mutex g_err_mutex;
static std::string g_last_error;

void set_global_error(const std::string& s) {
  std::lock_guard<std::mutex> lk(g_err_mutex);
  g_last_error = s;
}

int fail(r3d_ctx* ctx, int code, const std::string& msg) {
  // workers and batch tails report from several threads: the context's message is written under the same lock
  {
    std::lock_guard<std::mutex> lk(g_err_mutex);
    if (ctx) ctx->last_error = msg;
    g_last_error = msg;
  }
  return code;
}

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (PFN_encodeTiled)p;
  return fn;
}

void* pool_alloc(DeviceWorker& w, size_t bytes) {
  bytes = (bytes + 255) / 256 * 256;
  auto it = w.pool_free_blocks.lower_bound(bytes);
  if (it != w.pool_free_blocks.end() && it->first <= bytes + bytes / 4 + 4096) {
    void* p = it->second;
    w.pool_free_blocks.erase(it);
    return p;
  }
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    // give cached blocks back to the driver and retry once
    for (auto& kv : w.pool_free_blocks) { cudaFree(kv.second); w.pool_sizes.erase(kv.second); }
    w.pool_free_blocks.clear();
    if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
  }
  w.pool_sizes[p] = bytes;
  return p;
}

void pool_release(DeviceWorker& w, void* p) {
  if (!p) return;
  auto it = w.pool_sizes.find(p);
  if (it == w.pool_sizes.end()) { cudaFree(p); return; }
  w.pool_free_blocks.insert({it->second, p});
}

static void free_view(DeviceWorker& w, ViewDev& v) {
  pool_release(w, v.d_desc);
  pool_release(w, v.d_opQ);
  pool_release(w, v.d_opD);
  pool_release(w, v.d_norm);
  pool_release(w, v.d_xy);
  pool_release(w, v.d_stats);
  if (v.d_cascade) pool_release(w, v.d_cascade);
  v = ViewDev();
}

static void free_worker(DeviceWorker& w) {
  if (w.device < 0) return;
  cudaSetDevice(w.device);
  for (auto& kv : w.views) free_view(w, kv.second);
  w.views.clear();
  for (auto& kv : w.pool_sizes) cudaFree(kv.first);
  w.pool_sizes.clear();
  w.pool_free_blocks.clear();
  void* ptrs[] = {w.d_pairs, w.d_items, w.d_keys, w.d_fb, w.d_nn, w.d_tmapQ, w.d_tmapD,
                  w.d_cnt, w.d_slot, w.d_list, w.d_parts, w.d_list2, w.d_mdense, w.d_scan};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  for (auto& o : w.out) {
    if (o.d_matches) cudaFree(o.d_matches);
    if (o.d_counters) cudaFree(o.d_counters);
    if (o.h_counters) cudaFreeHost(o.h_counters);
    if (o.h_matches) cudaFreeHost(o.h_matches);
    if (o.h_stage) cudaFreeHost(o.h_stage);
    for (auto& e : o.ev)
      if (e) cudaEventDestroy(e);
  }
  for (void*& hp : w.h_fstage)
    if (hp) { cudaFreeHost(hp); hp = nullptr; }
  if (w.stream) cudaStreamDestroy(w.stream);
  if (w.copy_stream) cudaStreamDestroy(w.copy_stream);
  w = DeviceWorker();
}

// Encode the two TMA descriptors of a view: 2-D fp16 [n_pad][kp], box = 64 columns x 128 rows,
// 128-byte swizzle (the K-major SWIZZLE_128B operand layout of wgmma).  Integer path: two uint8 maps over the
// descriptors themselves, both with 128-column boxes (TMA zero-fills columns >= dim):
//   query role     2-D [n][dim], box 128 rows in natural order (rows >= n zero-filled)
//   database role  5-D (column, e, q, jj, g) with strides (1, D, 8 D, 2 D, 32 D) bytes, box {128, 2, 4, 4, 4}: database
//                  row 32 g + 8 q + 2 jj + e lands in shared-memory row 32 g + 8 jj + 2 q + e, a 4 x 4 transpose of
//                  row pairs inside every 32-row group, so that the accumulator columns of one lane of a wgmma quad
//                  are 8 consecutive database rows (k_l2_candidates.cu).  The map covers ceil(n / 32) whole groups:
//                  d_desc is padded to that many rows with zeros (r3d_upload_regions), later groups are zero-filled.
static int encode_view_maps(r3d_ctx* ctx, DeviceWorker& w, ViewDev& v, uint32_t slot) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return fail(ctx, R3D_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap maps[2];
  void* bases[2] = {(void*)v.d_opQ, (void*)v.d_opD};
  if (v.int_ops) {
    const cuuint64_t D = v.dim;
    cuuint64_t gdim[2] = {D, (cuuint64_t)std::max<uint32_t>(v.n, 1)};
    cuuint64_t gstride[1] = {D};
    cuuint32_t box[2] = {128, (cuuint32_t)kTileRows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&maps[0], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, v.d_desc, gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(ctx, R3D_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
    cuuint64_t gdim5[5] = {D, 2, 4, 4, (cuuint64_t)(int_desc_rows(v.n) / kGroupRows)};
    cuuint64_t gstride5[4] = {D, 8 * D, 2 * D, kGroupRows * D};
    cuuint32_t box5[5] = {128, 2, 4, 4, kTileRows / kGroupRows};
    cuuint32_t estr5[5] = {1, 1, 1, 1, 1};
    r = enc(&maps[1], CU_TENSOR_MAP_DATA_TYPE_UINT8, 5, v.d_desc, gdim5, gstride5, box5, estr5,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
      return fail(ctx, R3D_ERR_CUDA, "cuTensorMapEncodeTiled failed for the permuted database map: " + std::to_string((int)r));
  }
  for (int m = 0; m < 2 && !v.int_ops; ++m) {
    cuuint64_t gdim[2] = {(cuuint64_t)v.kp, (cuuint64_t)(v.tc_ok ? v.n_pad : (uint32_t)kRowPad)};
    cuuint64_t gstride[1] = {(cuuint64_t)v.kp * sizeof(__half)};
    cuuint32_t box[2] = {(cuuint32_t)kKBlock, (cuuint32_t)kTileRows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&maps[m], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, bases[m], gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(ctx, R3D_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  }
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(w.d_tmapQ + slot, &maps[0], sizeof(CUtensorMap), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(w.d_tmapD + slot, &maps[1], sizeof(CUtensorMap), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));  // maps[] is a stack temporary
  return R3D_OK;
}

static int ensure_tmap_capacity(r3d_ctx* ctx, DeviceWorker& w, uint32_t need) {
  if (need <= w.tmap_cap) return R3D_OK;
  uint32_t cap = w.tmap_cap ? w.tmap_cap : 64;
  while (cap < need) cap *= 2;
  CUtensorMap *nq = nullptr, *nd = nullptr;
  R3D_CUDA_TRY(ctx, cudaMalloc(&nq, cap * sizeof(CUtensorMap)));
  R3D_CUDA_TRY(ctx, cudaMalloc(&nd, cap * sizeof(CUtensorMap)));
  if (w.tmap_cap) {
    R3D_CUDA_TRY(ctx, cudaMemcpy(nq, w.d_tmapQ, w.tmap_cap * sizeof(CUtensorMap), cudaMemcpyDeviceToDevice));
    R3D_CUDA_TRY(ctx, cudaMemcpy(nd, w.d_tmapD, w.tmap_cap * sizeof(CUtensorMap), cudaMemcpyDeviceToDevice));
    cudaFree(w.d_tmapQ);
    cudaFree(w.d_tmapD);
  }
  w.d_tmapQ = nq;
  w.d_tmapD = nd;
  w.tmap_cap = cap;
  return R3D_OK;
}

// Bring every view of a worker to the "prepared" state (fp16 operands + error constants).
// Lazy: called by the first matching call after uploads.  One synchronisation for all views.
int prepare_views(r3d_ctx* ctx, DeviceWorker& w) {
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  std::vector<ViewDev*> fresh;
  for (auto& kv : w.views)
    if (!kv.second.prepared) fresh.push_back(&kv.second);
  if (fresh.empty()) return R3D_OK;
  for (ViewDev* v : fresh) {
    int rc = launch_view_stats(ctx, w, *v);
    if (rc) return rc;
  }
  std::vector<float> stats(4 * fresh.size());
  for (size_t i = 0; i < fresh.size(); ++i)
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(&stats[4 * i], fresh[i]->d_stats, 4 * sizeof(float), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  float max_n2 = 0.f;
  for (size_t i = 0; i < fresh.size(); ++i) {
    ViewDev* v = fresh[i];
    v->max_norm = std::sqrt(stats[4 * i + 0]) * (1.f + 1e-6f);
    v->max_hnorm = std::sqrt(stats[4 * i + 1]) * (1.f + 1e-6f);
    v->max_dnorm = std::sqrt(stats[4 * i + 2]) * (1.f + 1e-6f);
    v->max_abs = stats[4 * i + 3];
    if (v->int_ops) {  // the stats pass wrote its exact norms: nothing else to prepare, no part in e0
      v->prepared = true;
      continue;
    }
    // a view the fp16 operands cannot represent (|a_k| > 32000, or ||a||^2 >= 2^28 for the two-piece norm split)
    // keeps its exact descriptors only: its pairs take the exact scan (slower, same results)
    if (!v->tc_ok || !(v->max_abs <= 32000.f) || !(stats[4 * i + 0] < 2.6e8f)) {
      v->tc_ok = false;
      v->prepared = true;
      continue;
    }
    max_n2 = std::fmax(max_n2, stats[4 * i + 0]);
  }
  for (auto& kv : w.views)
    if (kv.second.prepared && kv.second.tc_ok && !kv.second.int_ops) max_n2 = std::fmax(max_n2, kv.second.max_norm * kv.second.max_norm);
  // Norm split scale: ||a||^2 ~= p0*2^e0 + p1*2^(e0-11) with p0 <= 2^13 and 2^(e0-11) a normal fp16.
  int e0 = -3;
  if (max_n2 > 0.f) {
    int ex;
    std::frexp(max_n2 * 1.0001f, &ex);  // max_n2 < 2^ex
    e0 = std::max(-3, ex - 13);
  }
  if (e0 > 15) e0 = 15;  // unreachable: norms that large were routed to the exact scan above
  if (w.e0_fixed && e0 < w.e0) e0 = w.e0;  // never shrink: keeps already prepared views valid
  const bool redo_all = w.e0_fixed && e0 != w.e0;
  w.e0 = e0;
  w.e0_fixed = true;
  for (auto& kv : w.views) {
    ViewDev& v = kv.second;
    if (!v.tc_ok || v.int_ops) continue;
    if (v.prepared && !redo_all) continue;
    int rc = launch_view_prepare(ctx, w, v, e0);
    if (rc) return rc;
    v.prepared = true;
    v.prepared_e0 = e0;
  }
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  return R3D_OK;
}

}  // namespace r3d

using namespace r3d;

extern "C" {

int r3d_abi_version(void) { return R3D_ABI_VERSION; }

const char* r3d_last_error(const r3d_ctx* ctx) {
  if (ctx) return ctx->last_error.c_str();
  static thread_local std::string copy;
  std::lock_guard<std::mutex> lk(g_err_mutex);
  copy = g_last_error;
  return copy.c_str();
}

int r3d_create(const int* device_ids, int n_devices, r3d_ctx** out) {
  if (!out) return fail(nullptr, R3D_ERR_INVALID, "r3d_create: out is NULL");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(nullptr, R3D_ERR_NO_DEVICE,
                std::string("r3d_create: no CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "count=0") +
                    "); libr3dgpu has no CPU fallback");
  std::vector<int> ids;
  if (device_ids && n_devices > 0) ids.assign(device_ids, device_ids + n_devices);
  else ids.push_back(0);
  r3d_ctx* ctx = new r3d_ctx();
  for (int id : ids) {
    if (id < 0 || id >= count) {
      delete ctx;
      return fail(nullptr, R3D_ERR_INVALID, "r3d_create: bad device id " + std::to_string(id));
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, id);
    if (prop.major != 9 || prop.minor != 0) {
      delete ctx;
      return fail(nullptr, R3D_ERR_NO_DEVICE,
                  "r3d_create: device " + std::to_string(id) + " is sm_" + std::to_string(prop.major) +
                      std::to_string(prop.minor) + "; this library is built for sm_90a only");
    }
    DeviceWorker w;
    w.device = id;
    w.sm_count = prop.multiProcessorCount;
    cudaSetDevice(id);
    if (cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&w.copy_stream, cudaStreamNonBlocking) != cudaSuccess) {
      delete ctx;
      return fail(nullptr, R3D_ERR_CUDA, "r3d_create: stream / counter allocation failed");
    }
    ctx->workers.push_back(w);
  }
  ctx->host_threads = (int)std::thread::hardware_concurrency();
  if (ctx->host_threads < 1) ctx->host_threads = 1;
  if (ctx->host_threads > 64) ctx->host_threads = 64;
  *out = ctx;
  return R3D_OK;
}

void r3d_destroy(r3d_ctx* ctx) {
  if (!ctx) return;
  r3d_comm_destroy(ctx);
  for (auto& w : ctx->workers) free_worker(w);
  delete ctx;
}

int r3d_clear_regions(r3d_ctx* ctx) {
  if (!ctx) return R3D_ERR_INVALID;
  for (auto& w : ctx->workers) {
    cudaSetDevice(w.device);
    cudaStreamSynchronize(w.stream);
    for (auto& kv : w.views) free_view(w, kv.second);
    w.views.clear();
    w.view_slot.clear();
    w.e0_fixed = false;
    w.e0 = -3;
  }
  return R3D_OK;
}

int r3d_upload_regions(r3d_ctx* ctx, uint32_t view_id, const void* desc, uint32_t n, uint32_t dim, int dtype,
                       const float* xy) {
  if (!ctx) return R3D_ERR_INVALID;
  if (dtype != R3D_F32 && dtype != R3D_U8) return fail(ctx, R3D_ERR_INVALID, "r3d_upload_regions: bad dtype");
  if (n > 0 && (!desc || dim == 0)) return fail(ctx, R3D_ERR_INVALID, "r3d_upload_regions: NULL descriptors");
  for (auto& w : ctx->workers) {
    R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
    auto it = w.views.find(view_id);
    if (it != w.views.end()) {
      R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
      free_view(w, it->second);
      w.views.erase(it);
    }
    ViewDev v;
    v.n = n; v.dim = dim; v.dtype = (uint32_t)dtype;
    v.n_pad = (uint32_t)pad_up((int)(n ? n : 1), kRowPad);
    v.int_ops = int_operand(dtype, dim);
    // fp16: Kp <= 256 columns, and the exact re-rank reads whole 4-byte words of a row; wider descriptors and uint8 rows
    // of D % 4 != 0 bytes are matched by the exact scan only
    v.tc_ok = v.int_ops || (dim <= 240 && (dtype == R3D_F32 || dim % 4 == 0));
    v.kp = v.int_ops ? 0u : (uint32_t)operand_cols((int)(dim && v.tc_ok ? dim : 16));
    const size_t rb = dtype == R3D_F32 ? (size_t)dim * 4 : (size_t)dim;
    // >= one row: the extent of the u8 maps; integer path: whole 32-row groups of the permuted database map
    const uint32_t desc_rows = v.int_ops ? int_desc_rows(n) : std::max<uint32_t>(n, 1);
    v.d_desc = pool_alloc(w, std::max<size_t>(rb * desc_rows, 16));
    if (v.int_ops) {
      v.d_norm = (int32_t*)pool_alloc(w, (size_t)v.n_pad * sizeof(int32_t));
    } else {
      const size_t op_rows = v.tc_ok ? v.n_pad : (uint32_t)kRowPad;  // a token block keeps the tensor maps valid
      v.d_opQ = (__half*)pool_alloc(w, op_rows * v.kp * sizeof(__half));
      v.d_opD = (__half*)pool_alloc(w, op_rows * v.kp * sizeof(__half));
    }
    v.d_stats = (float*)pool_alloc(w, 4 * sizeof(float));
    if (xy && n) v.d_xy = (float2*)pool_alloc(w, (size_t)n * sizeof(float2));
    if (!v.d_desc || (v.int_ops ? !v.d_norm : (!v.d_opQ || !v.d_opD)) || !v.d_stats || (xy && n && !v.d_xy)) {
      free_view(w, v);
      return fail(ctx, R3D_ERR_NOMEM, "r3d_upload_regions: device allocation failed");
    }
    // every error exit below returns the view's device blocks to the pool
    struct ViewGuard {
      DeviceWorker& w; ViewDev& v; bool armed = true;
      ~ViewGuard() { if (armed) { cudaStreamSynchronize(w.stream); free_view(w, v); } }
    } guard{w, v};
    if (n) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(v.d_desc, desc, rb * n, cudaMemcpyHostToDevice, w.stream));
    if (v.int_ops && desc_rows > n)  // the database map reads these rows: zeros, so that padding keys are kPadNorm + ||q||^2
      R3D_CUDA_TRY(ctx, cudaMemsetAsync((char*)v.d_desc + rb * n, 0, rb * (desc_rows - n), w.stream));
    if (xy && n) {
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(v.d_xy, xy, (size_t)n * sizeof(float2), cudaMemcpyHostToDevice, w.stream));
      v.h_xy.assign(xy, xy + 2 * (size_t)n);
      v.has_xy = true;
    }
    ctx->pending_h2d += rb * n + (xy ? (size_t)n * 8 : 0);
    uint32_t slot;
    auto sit = w.view_slot.find(view_id);
    const bool new_slot = sit == w.view_slot.end();
    slot = new_slot ? (uint32_t)w.view_slot.size() : sit->second;
    int rc = ensure_tmap_capacity(ctx, w, slot + 1);
    if (rc) return rc;
    rc = encode_view_maps(ctx, w, v, slot);  // synchronises the stream: host buffers are consumed
    if (rc) return rc;
    if (new_slot) w.view_slot[view_id] = slot;  // only a stored view keeps a slot
    guard.armed = false;
    w.views[view_id] = std::move(v);
  }
  return R3D_OK;
}

int r3d_debug_view_operands(r3d_ctx* ctx, uint32_t view_id, uint32_t* n_pad, uint32_t* kp, uint16_t* opQ, uint16_t* opD,
                            float* stats, int* e0) {
  if (!ctx || !n_pad || !kp || ctx->workers.empty()) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_view_operands: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  int rc = prepare_views(ctx, w);  // as the next matching call would
  if (rc) return rc;
  auto it = w.views.find(view_id);
  if (it == w.views.end()) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_view_operands: unknown view");
  const ViewDev& v = it->second;
  *n_pad = v.n_pad;
  *kp = (v.tc_ok && !v.int_ops) ? v.kp : 0u;
  const size_t halves = (size_t)*n_pad * *kp;
  if (opQ && halves) R3D_CUDA_TRY(ctx, cudaMemcpy(opQ, v.d_opQ, halves * sizeof(__half), cudaMemcpyDeviceToHost));
  if (opD && halves) R3D_CUDA_TRY(ctx, cudaMemcpy(opD, v.d_opD, halves * sizeof(__half), cudaMemcpyDeviceToHost));
  if (stats) R3D_CUDA_TRY(ctx, cudaMemcpy(stats, v.d_stats, 4 * sizeof(float), cudaMemcpyDeviceToHost));
  if (e0) *e0 = w.e0;
  return R3D_OK;
}

int r3d_get_match_timing(const r3d_ctx* ctx, r3d_match_timing* out) {
  if (!ctx || !out) return R3D_ERR_INVALID;
  *out = ctx->match_timing;
  return R3D_OK;
}

int r3d_get_filter_timing(const r3d_ctx* ctx, r3d_filter_timing* out) {
  if (!ctx || !out) return R3D_ERR_INVALID;
  *out = ctx->filter_timing;
  return R3D_OK;
}

}  // extern "C"
