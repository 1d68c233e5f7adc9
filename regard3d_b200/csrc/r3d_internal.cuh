// r3d_internal.cuh -- internal declarations of libr3dgpu (H100 / sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <chrono>
#include <functional>
#include <map>
#include <mutex>
#include <thread>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/r3dgpu.h"
#include "r3d_matches.h"

// ------------------------------------------------------------------------------------------------
// Geometry of the tensor-core candidate kernel (k_l2_candidates.cu) and the operand layout.
// ------------------------------------------------------------------------------------------------
namespace r3d {

constexpr int kTileRows = 128;      // rows of one TMA box; query rows per work item of the fp16 path
constexpr int kKBlock = 64;         // fp16 elements per 128-byte swizzle row
constexpr int kQB = 2;              // integer path: 128-row query boxes per work item
constexpr int kSuperRows = kTileRows * kQB;  // query rows per work item of the integer path
constexpr int kRowPad = 256;        // every view is padded to a multiple of this many rows
constexpr int kBiasCols = 16;       // one MMA K-step holding the norm terms
#ifndef R3D_CHUNK
#define R3D_CHUNK 8
#endif
constexpr int kChunk = R3D_CHUNK;   // database columns summarised by one candidate key (8, or 16 as a build-time A/B)
constexpr int kChunkBits = 13;      // max low mantissa bits of a key that hold the chunk id
constexpr int kNumKeys = 6;         // keys kept per query (5 candidate chunks + 1 bound)
constexpr int kKeyStride = 8;       // uint32 per query row in the key array (two 16-byte stores)
constexpr int kMaxKBlocks = 4;      // Kp <= 256  (descriptor dim <= 240)
constexpr uint32_t kMaxDbRowsTC = (1u << kChunkBits) * kChunk;  // 65536

inline int pad_up(int x, int m) { return (x + m - 1) / m * m; }
int operand_col_align();  // 16, or 64 (R3D_KP_ALIGN) to make operand rows 128-byte aligned
inline int operand_ksteps(int dim) { return (pad_up(dim, 16) + kBiasCols) / 16; }
inline int operand_cols(int dim) { return pad_up(pad_up(dim, 16) + kBiasCols, operand_col_align()); }  // Kp
// uint8 descriptors whose rows are whole 16-byte TMA strides take the integer tensor-core path: the candidate kernel
// reads d_desc directly and computes exact squared distances (u8 x u8 -> s32 wgmma), no fp16 operands
inline bool int_operand(int dtype, uint32_t dim) { return dtype == R3D_U8 && dim > 0 && dim % 16 == 0 && dim <= 256; }
constexpr int32_t kPadNorm = 1 << 28;  // ||a||^2 of a padding row of the integer path: above every real distance
                                       // (< 2^24 for dim <= 256), and no epilogue sum reaches 2^31
constexpr uint32_t kGroupRows = 32;    // integer path: database rows permuted together by the database tensor map
// rows of d_desc on the integer path: whole groups of the database map (zeros beyond n), at least one
inline uint32_t int_desc_rows(uint32_t n) { return (std::max<uint32_t>(n, 1) + kGroupRows - 1) / kGroupRows * kGroupRows; }
// query rows per work item of the candidate kernel (a divisor of kRowPad)
inline uint32_t item_rows(int dtype, uint32_t dim) { return int_operand(dtype, dim) ? kSuperRows : kTileRows; }

struct ViewDev {
  uint32_t n = 0, dim = 0, dtype = 0, n_pad = 0, kp = 0;
  void* d_desc = nullptr;    // original descriptors [n][dim] (f32 or u8): exact re-rank operand
                             // (integer path: zero rows up to int_desc_rows(n))
  __half* d_opQ = nullptr;   // query-role operand    [n_pad][kp]: -2*b | S0 S1 q0 q1 0...
  __half* d_opD = nullptr;   // database-role operand [n_pad][kp]:    a  | p0 p1 S0 S1 0...
  int32_t* d_norm = nullptr; // integer path: exact ||a||^2 [n_pad], kPadNorm on padding rows
  bool int_ops = false;      // int_operand(dtype, dim): no d_opQ / d_opD, kp = 0
  float2* d_xy = nullptr;    // positions [n]
  std::vector<float> h_xy;   // host copy (coordinate de-duplication, RANSAC set-up)
  std::vector<uint32_t> h_yrank;   // build_view_ranks(): tables of the descent-free coordinate de-duplication
  std::vector<uint8_t> h_xshared;
  uint32_t n_slots = 0;
  bool ranks_tried = false;  // tables stay empty for views with non-finite positions (classic replay then)
  bool has_xy = false;
  bool prepared = false;
  bool tc_ok = true;         // false: no fp16 operands (dim > 240 or values outside the fp16 operand range):
                             // pairs touching this view are matched by the exact CUDA-core scan only
  int prepared_e0 = 0;
  // error-bound constants (host copies of device reductions)
  float max_norm = 0.f;      // max_i ||a_i||
  float max_hnorm = 0.f;     // max_i ||fp16(a_i)||
  float max_dnorm = 0.f;     // max_i ||a_i - fp16(a_i)||
  float max_abs = 0.f;       // max |a_ik|
  float* d_stats = nullptr;  // 4 floats: max n2, max hn2, max dn2, max abs
  // cascade hashing (cascade.cu): one block holding hash codes, bucket offsets / ids, bucket ids of this view
  void* d_cascade = nullptr;
  size_t cascade_bytes = 0;
  uint64_t cascade_epoch = 0;   // the zero-mean epoch the tables were hashed under
  uint32_t cascade_index = 0;   // row of the worker's CascadeView table
};

struct CascadeView {            // device-visible tables of one hashed view
  uint32_t* code;               // [n][words] sign bits of the primary projections
  uint16_t* bucket;             // [n][6] bucket id per group
  uint32_t* bk_ofs;             // [6][1025] bucket offsets
  uint32_t* bk_ids;             // [6][n] descriptor ids, ascending inside a bucket
  uint32_t n, words;
};

struct PairDesc {            // one entry per pair of a batch (device + host)
  uint32_t I, J;             // view ids
  uint32_t nI, nJ;           // feature counts
  uint32_t nI_pad, nJ_pad;
  uint32_t q_ofs;            // first row of this pair in the per-batch key / nn arrays
  uint32_t use_tc;           // 1: tensor-core candidates available, 0: exact scan only
  float eps_abs;             // absolute error bound of a candidate value vs the real-valued distance
  uint32_t slotI, slotJ;     // tensor-map slots of the two views
  uint32_t chunk_bits;       // low mantissa bits of a key that hold the chunk id (<= kChunkBits)
  const void* descI;         // original descriptors of I / J (device)
  const void* descJ;
  const int32_t* normI;      // integer path: exact squared norms of I / J (ViewDev::d_norm), else null
  const int32_t* normJ;
};
static_assert(sizeof(PairDesc) == 80, "PairDesc layout");

struct WorkItem { uint32_t pair; uint32_t sb; };  // sb: query block (item_rows() rows) index

constexpr uint32_t kCounterWords = 16 + 4096;  // 16 scalar counters + one match counter per pair of the batch
struct OutSlot {  // double-buffered outputs of a matching batch
  void* d_matches = nullptr; size_t matches_cap = 0;  // packed (i, j) of the batch, bucketed by pair
  uint32_t* d_counters = nullptr;  // [1] exact-scan list, [3] stage C, [4] deferred by stage A, [16 + k] matches of pair k
  uint32_t* h_counters = nullptr;  // pinned
  void* h_matches = nullptr; size_t h_matches_cap = 0;  // pinned
  void* h_stage = nullptr; size_t h_stage_cap = 0;      // pinned: PairDesc[] + WorkItem[] of the batch (a pageable
                                                        // source would make the "async" upload wait for the stream)
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
};

struct DeviceWorker {
  int device = -1;
  int sm_count = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  std::map<uint32_t, ViewDev> views;
  // tensor maps, indexed by view slot
  std::map<uint32_t, uint32_t> view_slot;
  CUtensorMap* d_tmapQ = nullptr;
  CUtensorMap* d_tmapD = nullptr;
  uint32_t tmap_cap = 0;
  // per-context scale exponent of the norm split (S0 = 2^e0, S1 = 2^(e0-11))
  int e0 = -3;
  bool e0_fixed = false;
  // scratch (grown on demand)
  void* d_pairs = nullptr; size_t pairs_cap = 0;
  void* d_items = nullptr; size_t items_cap = 0;
  void* d_keys = nullptr; size_t keys_cap = 0;
  OutSlot out[2];
  // size-bucketed cache of device blocks released by r3d_clear_regions / re-uploads: cudaMalloc and
  // cudaFree synchronise the device and cost ~ms, the upload path must not pay them per view
  std::multimap<size_t, void*> pool_free_blocks;
  std::map<void*, size_t> pool_sizes;
  void* d_fb = nullptr; size_t fb_cap = 0;
  void* d_nn = nullptr; size_t nn_cap = 0;
  void* d_cnt = nullptr; size_t cnt_cap = 0;      // binned re-rank scratch
  void* d_slot = nullptr; size_t slot_cap = 0;
  void* d_list = nullptr; size_t list_cap = 0;
  void* d_parts = nullptr; size_t parts_cap = 0;
  void* d_list2 = nullptr; size_t list2_cap = 0;
  void* d_mdense = nullptr; size_t mdense_cap = 0;
  void* d_scan = nullptr; size_t scan_cap = 0;      // split exact scan: partial top-2s + arrival counters  // (i, j) per pair segment, before packing
  void* h_fstage[2] = {nullptr, nullptr}; size_t h_fstage_cap = 0;  // pinned staging of the filter's result download
  r3d_match_timing timing{};  // per-worker accumulation (summed into the context after a call)
  // cascade hashing: projection table [dim][dim + 60], the hashed views' table, the epoch they belong to
  float* d_cascade_proj = nullptr;
  uint32_t cascade_dim = 0;
  CascadeView* d_cascade_views = nullptr;
  uint64_t cascade_epoch = 0;
};

}  // namespace r3d


struct r3d_ctx {
  std::vector<r3d::DeviceWorker> workers;
  std::string last_error;
  r3d_match_timing match_timing{};
  uint64_t pending_h2d = 0;  // bytes uploaded since the last matching call
  r3d_filter_timing filter_timing{};
  r3d_relpose_timing relpose_timing{};
  r3d_resection_timing resection_timing{};
  r3d_akaze_timing akaze_timing{};
  r3d_extract_timing extract_timing{};
  int host_threads = 0;
  // optional NCCL communicator (comm.cu): only the bundle adjustment exchanges data between ranks
  void* nccl_comm = nullptr;
  int comm_world = 1, comm_rank = 0;
  uint64_t cascade_epoch_counter = 0;
};

namespace r3d {

void set_global_error(const std::string& s);
int fail(r3d_ctx* ctx, int code, const std::string& msg);

// comm.cu: in-place all-reduce of `n` doubles on the worker's stream; no-op without a communicator
enum CommOp { kCommSum = 0, kCommMax = 2 };
int comm_allreduce(r3d_ctx* ctx, cudaStream_t stream, double* buf, size_t n, CommOp op);

#define R3D_CUDA_TRY(ctx, call)                                                            \
  do {                                                                                     \
    cudaError_t _e = (call);                                                               \
    if (_e != cudaSuccess)                                                                 \
      return r3d::fail((ctx), R3D_ERR_CUDA,                                                \
                       std::string(#call) + ": " + cudaGetErrorString(_e) + " (" +         \
                           __FILE__ + ":" + std::to_string(__LINE__) + ")");               \
  } while (0)

template <typename T>
int ensure_capacity(r3d_ctx* ctx, void** p, size_t* cap, size_t need_elems) {
  const size_t need = need_elems * sizeof(T);
  if (*cap >= need && *p) return R3D_OK;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  size_t alloc = need + need / 4 + 256;
  cudaError_t e = cudaMalloc(p, alloc);
  if (e != cudaSuccess) return fail(ctx, R3D_ERR_NOMEM, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  *cap = alloc;
  return R3D_OK;
}

// dense Cholesky + both triangular solves of an SPD system on the worker's stream (ba.cu: the cooperative k_chol_fused,
// one CTA per SM).  A: (n+1) x n row-major, the system with its right-hand side as row n, overwritten; L: (n+1) x n + 64,
// receives the lower factor (row n: the forward-substituted rhs); Linv: ceil(n / kCholNB) inverses of the kCholNB x kCholNB
// diagonal blocks of L; *flag (zeroed by the caller) becomes 1 when A is not positive definite; x: n, the solution.
// Only the lower triangle of A is read.  grid: CTAs of the cooperative launch, 0 = one per SM (R3D_ERR_INVALID beyond
// what can be co-resident); the result does not depend on it.
constexpr int kCholNB = 32;
int dense_cholesky(r3d_ctx* ctx, DeviceWorker& w, double* A, double* L, double* Linv, int n, double* flag, double* x, int grid = 0);
int dense_cholesky_grid(r3d_ctx* ctx, DeviceWorker& w, int* grid);  // resolves grid 0, checks co-residency
// the same with the envelope kernel (ba.cu: k_chol_envelope on ONE cluster of `ctas` = 1..8 CTAs, R3D_ERR_INVALID
// otherwise or for an odd n).  A and L: (n+1) x n + 64 (the slack is read, never used); ft (device): first column tile
// of each of the ceil((n+1) / kCholNB) row tiles, every panel at most 24 active row tiles (the caller checks); no Linv.
int envelope_cholesky(r3d_ctx* ctx, DeviceWorker& w, double* A, double* L, int n, const int* ft, int ctas, double* flag, double* x);

int prepare_views(r3d_ctx* ctx, DeviceWorker& w);
void* pool_alloc(DeviceWorker& w, size_t bytes);  // nullptr on failure
void pool_release(DeviceWorker& w, void* p);

// device scratch out of the worker's size-bucketed pool: no cudaMalloc / cudaFree per call -- both synchronise the
// device and cost up to a second per call on multi-GPU boxes.  Everything that touches these blocks is ordered on
// w.stream, so a released block may be handed out again at once.  alloc(n): max(n, 1) elements, false when the pool
// cannot provide them; a second alloc releases the earlier block.
template <typename T>
struct DevArr {
  DeviceWorker* w;
  T* p = nullptr;
  explicit DevArr(DeviceWorker& worker) : w(&worker) {}
  DevArr(const DevArr&) = delete;
  DevArr& operator=(const DevArr&) = delete;
  ~DevArr() { pool_release(*w, p); }
  bool alloc(size_t n) {
    pool_release(*w, p);
    p = (T*)pool_alloc(*w, std::max<size_t>(n, 1) * sizeof(T));
    return p != nullptr;
  }
};

// N CUDA events, destroyed with the object; create(false): ordering only (cudaEventDisableTiming)
template <int N>
struct Events {
  cudaEvent_t e[N] = {};
  Events() = default;
  Events(const Events&) = delete;
  Events& operator=(const Events&) = delete;
  ~Events() {
    for (cudaEvent_t x : e)
      if (x) cudaEventDestroy(x);
  }
  cudaError_t create(bool timing = true) {
    for (cudaEvent_t& x : e) {
      const cudaError_t r = cudaEventCreateWithFlags(&x, timing ? cudaEventDefault : cudaEventDisableTiming);
      if (r != cudaSuccess) return r;
    }
    return cudaSuccess;
  }
  float ms(int a, int b) const {  // elapsed time between two recorded timing events
    float t = 0.f;
    cudaEventElapsedTime(&t, e[a], e[b]);
    return t;
  }
};

inline double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Independent work items [0, n) spread over `parts` devices: cut[k] .. cut[k + 1] is part k, contiguous ranges of equal
// sums of weight(i) + 1 (prefix sums, then lower_bound on k / parts of the total).
template <typename Weight>
std::vector<uint64_t> balanced_cuts(uint64_t n, size_t parts, Weight weight) {
  std::vector<uint64_t> cut(parts + 1, 0);
  cut[parts] = n;
  if (parts < 2) return cut;
  std::vector<double> cost(n + 1, 0.0);
  for (uint64_t i = 0; i < n; ++i) cost[i + 1] = cost[i] + (double)weight(i) + 1.0;
  for (size_t k = 1; k < parts; ++k)
    cut[k] = std::min<uint64_t>(n, (uint64_t)(std::lower_bound(cost.begin(), cost.end(), cost[n] * (double)k / (double)parts) - cost.begin()));
  return cut;
}

// fn(k, worker k) for every worker of the context: inline for a single worker, otherwise on one thread per worker.
// Returns the first non-zero return code in worker order.
template <typename Fn>
int fan_out(r3d_ctx* ctx, Fn&& fn) {
  const size_t nw = ctx->workers.size();
  std::vector<int> rcs(nw, R3D_OK);
  if (nw == 1) {
    rcs[0] = fn((size_t)0, ctx->workers[0]);
  } else {
    std::vector<std::thread> th;
    for (size_t k = 0; k < nw; ++k) th.emplace_back([&, k]() { rcs[k] = fn(k, ctx->workers[k]); });
    for (auto& t : th) t.join();
  }
  for (int rc : rcs)
    if (rc) return rc;
  return R3D_OK;
}

// dynamic-scheduling parallel loop on the persistent host pool (host_pool.cpp); n_threads bounds the
// concurrency of THIS loop (the caller counts as one)
void pool_parallel_for(int n_threads, size_t n, const std::function<void(size_t)>& f);
template <typename F>
inline void parallel_for(int n_threads, size_t n, F&& f) {
  if (n == 0) return;
  if (n_threads <= 1 || n == 1) {
    for (size_t i = 0; i < n; ++i) f(i);
    return;
  }
  const std::function<void(size_t)> fn = [&f](size_t i) { f(i); };
  pool_parallel_for(n_threads, n, fn);
}

// ---- kernels (defined in the .cu files) --------------------------------------------------------
// operand preparation
int launch_view_stats(r3d_ctx* ctx, DeviceWorker& w, ViewDev& v);
int launch_view_prepare(r3d_ctx* ctx, DeviceWorker& w, ViewDev& v, int e0);
// tensor-core candidate kernel: persistent CTAs (TMA + wgmma); work items are 128-query blocks.  The operand kind
// (fp16 operands or the integer path) follows from dtype and dim, which every pair of a call shares.
int launch_l2_candidates(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const WorkItem* d_items,
                         uint32_t n_items, uint32_t* d_keys, int dtype, uint32_t dim);
// exact re-rank + ratio
int launch_rerank_list(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const uint32_t* d_keys, const void* d_parts,
                       const uint2* d_list, const uint32_t* d_list_count, uint32_t max_list, uint32_t dim, int dtype,
                       float ratio2, uint32_t* d_counters, uint2* d_matches, uint2* d_fallback, float4* d_nn);
// binned stage A (rerank_binned.cu); cstride = max chunks per pair + 1
int launch_rerank_binned(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, uint32_t n_pairs, uint32_t max_nJ,
                         uint32_t cstride, const uint32_t* d_keys, uint32_t dim, int dtype, float ratio2,
                         uint32_t* d_cnt, uint32_t* d_slot, uint32_t* d_list, void* d_parts, uint32_t* d_counters,
                         uint2* d_matches, uint2* d_list2, uint2* d_fallback, float4* d_nn);
// exact scan of listed queries
int launch_pack_matches(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, uint32_t n_pairs, const uint32_t* d_pair_cnt,
                        const uint2* d_dense, uint2* d_packed);
int launch_exact_scan(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const uint2* d_list,
                      const uint32_t* d_list_count, uint32_t max_list, uint32_t dim, int dtype,
                      float ratio2, uint32_t* d_counters, uint2* d_matches, float4* d_nn);
int launch_fill_all_queries(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, uint32_t n_pairs,
                            uint2* d_list, uint32_t* d_list_count);

// host post-processing (match_post.cpp)
size_t post_process_pair(r3d_indmatch* m, size_t n, const float* xyI, const float* xyJ,
                       bool coord_dedup);
constexpr int kPostLanes = 4;  // pairs one host thread advances in lockstep (independent trees hide each other's latency)
struct ViewRankRef { const uint32_t* yrank; const uint8_t* xshared; uint32_t n_slots; };
void build_view_ranks(const float* xy, uint32_t n, std::vector<uint32_t>& yrank, std::vector<uint8_t>& xshared,
                      uint32_t* n_slots);
void post_process_pairs(int lanes, r3d_indmatch* const* ms, size_t* counts, const float* const* xyIs, const float* const* xyJs,
                        bool coord_dedup, const ViewRankRef* ranks);

// r3d_save_features without the argument checks (features_io.cpp): nullptr, or the path that could not be written
const char* save_features(const char* feat_path, const char* desc_path, const float* xyso, const float* desc, uint64_t n,
                          uint32_t dim);

// LIOP-144 (liop.cu), shared by r3d_liop_describe and r3d_extract_features (akaze.cu)
namespace liop {
constexpr int kDim = 144, kMaxSlots = 16;
struct Tables;
struct Slots {  // by value: keypoints first[s] .. first[s + 1] - 1 sample image s (img[s], w[s] x h[s], row-major)
  const float* img[kMaxSlots];
  int w[kMaxSlots], h[kMaxSlots];
  uint32_t first[kMaxSlots + 1];
  int n;
};
// the inverse affine map of one keypoint (host, libm cos / sin): 6 floats
void affine_of(float x, float y, float kp_size, float kp_angle, float factor, float* M);
// the sampling tables in a pool block of w, uploaded on st; nullptr on failure
Tables* tables_to_device(DeviceWorker& w, cudaStream_t st);
// k_liop on st: one CTA per keypoint, d_M n x 6, d_desc n x kDim
int describe(r3d_ctx* ctx, cudaStream_t st, const Slots& S, const float* d_M, uint32_t n, const Tables* d_T, float* d_desc);
}  // namespace liop

// driver entry points
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

}  // namespace r3d
