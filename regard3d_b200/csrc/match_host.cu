// match_host.cu -- host orchestration of putative matching.
//
// r3d_match_pairs replaces Matcher_Regions(fDistRatio, BRUTE_FORCE_L2)::Match
// (src/R3DComputeMatches.cpp:2039, :2048; loop shape :437-488).  The reference's "serial I,
// omp-dynamic J, critical insert" becomes: all pairs of a batch in ONE persistent tensor-core
// launch (work item = pair x 256-query super-block), one re-rank launch, one exact-scan launch for
// the uncertified remainder, one compacted device->host copy, host de-duplication on a thread pool.
#include "r3d_internal.cuh"
#include "r3d_cascade.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <future>
#include <map>
#include <set>
#include <memory>
#include <mutex>
#include <thread>

namespace r3d {

namespace {

struct BatchPair {
  uint64_t src_index;  // index in the caller's pair list
  PairDesc pd;
};

// e0: the worker's norm-split exponent the views were prepared under (prepare_views runs first)
float pair_eps(const ViewDev& vi, const ViewDev& vj, int e0) {
  if (vi.int_ops && vj.int_ops) return 0.f;  // integer path: exact keys (the chunk-id packing is covered by pack_rel)
  const double nI = vi.max_norm, nJ = vj.max_norm;
  double e = 2.0 * ((double)vi.max_dnorm * nJ + (double)vi.max_hnorm * (double)vj.max_dnorm);
  // two-piece fp16 split of the squared norms: per row 2^-22 ||a||^2 while p0, p1 are normal, plus at most 2^(e0-36)
  // when they are fp16 subnormals (a row far smaller than the largest norm of the worker's views)
  e += std::ldexp(nI * nI + nJ * nJ, -21) + std::ldexp(1.0, e0 - 35);
  // fp32 accumulation inside the tensor core: measured on H100 up to 2^-22 (nI + nJ)^2 per k16 step (products aligned to
  // the running sum lose up to a quarter ulp each); twice that per step, and never less than 2^-18 (nI + nJ)^2
  e += std::ldexp((double)std::max(8, operand_ksteps((int)vi.dim)) * (nI + nJ) * (nI + nJ), -21);
  e *= 1.001;
  return (float)e + 1e-30f;
}

}  // namespace

// ---- result slabs ------------------------------------------------------------------------------------
// Every batch hands its de-duplicated matches over in one buffer that the returned r3d_matches keeps alive.
// Allocating these (3 MB each at C2, mmap-sized) afresh on every call made every other call 15-25 ms slower
// (page faults + munmap under the process-wide mm lock, with 30+ host threads running): buffers are recycled
// through a bounded process-wide free list instead; the shared_ptr deleter returns them.
namespace {
struct SlabPool {
  std::mutex mu;
  std::multimap<size_t, r3d_indmatch*> free_list;  // capacity (elements) -> buffer
  size_t cached_bytes = 0;
  static constexpr size_t kMaxCachedBytes = (size_t)2 << 30;
  r3d_indmatch* take(size_t n, size_t* cap) {
    {
      std::lock_guard<std::mutex> lk(mu);
      auto it = free_list.lower_bound(n);
      if (it != free_list.end() && it->first <= 2 * n + 4096) {
        r3d_indmatch* p = it->second;
        *cap = it->first;
        cached_bytes -= it->first * sizeof(r3d_indmatch);
        free_list.erase(it);
        return p;
      }
    }
    *cap = n + n / 4 + 1024;
    return new r3d_indmatch[*cap];  // not zero-filled
  }
  void give(r3d_indmatch* p, size_t cap) {
    {
      std::lock_guard<std::mutex> lk(mu);
      if (cached_bytes + cap * sizeof(r3d_indmatch) <= kMaxCachedBytes) {
        free_list.insert({cap, p});
        cached_bytes += cap * sizeof(r3d_indmatch);
        return;
      }
    }
    delete[] p;
  }
};
SlabPool& slab_pool() {
  static SlabPool* p = new SlabPool();  // leaked on purpose: results may outlive static destruction order
  return *p;
}
r3d_slab acquire_slab(size_t n, r3d_indmatch** out) {
  size_t cap = 0;
  r3d_indmatch* p = slab_pool().take(std::max<size_t>(n, 1), &cap);
  *out = p;
  return r3d_slab((void*)p, [cap](void* q) { slab_pool().give((r3d_indmatch*)q, cap); });
}
}  // namespace


// Runs the device pipeline for a list of pairs on one worker.
//  results[k]   : matches of pairs[k] (empty if none)
//  nn_out       : optional, for r3d_search_neighbours (single pair): float4 per query
static int match_on_worker(r3d_ctx* ctx, DeviceWorker& w, const uint32_t* pairs, uint64_t n_pairs, float ratio,
                           uint32_t flags, std::vector<r3d_span>& results, std::vector<r3d_slab>& slabs,
                           std::vector<float4>* nn_out, std::vector<uint4>* keys_dbg = nullptr) {
  const double t_enter = now_ms();
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  int rc = prepare_views(ctx, w);
  if (rc) return rc;
  results.assign(n_pairs, r3d_span{});
  std::mutex slab_mutex;
  const float ratio2 = ratio * ratio;  // Square(fDistRatio): b_squared_metric = true for BRUTE_FORCE_L2
  const bool want_matches = (nn_out == nullptr);
  const bool cascade = want_matches && (flags & R3D_MATCH_CASCADE_HASHING) != 0;  // CASCADE_HASHING_L2 (cascade.cu)

  // ---- build pair descriptors --------------------------------------------------------------
  std::vector<BatchPair> all;
  all.reserve(n_pairs);
  uint32_t dim = 0;
  int dtype = -1;
  for (uint64_t p = 0; p < n_pairs; ++p) {
    const uint32_t I = pairs[2 * p], J = pairs[2 * p + 1];
    auto iI = w.views.find(I), iJ = w.views.find(J);
    if (iI == w.views.end() || iJ == w.views.end())
      return fail(ctx, R3D_ERR_INVALID, "r3d_match_pairs: view " + std::to_string(iI == w.views.end() ? I : J) + " was not uploaded");
    const ViewDev& vi = iI->second;
    const ViewDev& vj = iJ->second;
    // reference: skip when either side has no regions (R3DComputeMatches.cpp:444-447, :471-475);
    // SearchNeighbours returns false when NN(2) > #database rows.
    if (vi.n < 2 || vj.n == 0) continue;  // (cascade hashing: fewer than 3 candidates -> no result either)
    if (vi.dim != vj.dim || vi.dtype != vj.dtype) continue;  // Type_id() mismatch -> skipped
    if (dtype < 0) { dim = vi.dim; dtype = (int)vi.dtype; }
    if (vi.dim != dim || (int)vi.dtype != dtype)
      return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_match_pairs: mixed descriptor types in one call");
    BatchPair bp;
    bp.src_index = p;
    PairDesc& pd = bp.pd;
    std::memset(&pd, 0, sizeof(pd));
    pd.I = I; pd.J = J; pd.nI = vi.n; pd.nJ = vj.n; pd.nI_pad = vi.n_pad; pd.nJ_pad = vj.n_pad;
    pd.slotI = w.view_slot[I]; pd.slotJ = w.view_slot[J];
    pd.descI = vi.d_desc; pd.descJ = vj.d_desc;
    pd.normI = vi.d_norm; pd.normJ = vj.d_norm;
    pd.use_tc = (!cascade && (flags & R3D_MATCH_EXACT_SCAN) == 0 && vi.tc_ok && vj.tc_ok && vi.n_pad <= kMaxDbRowsTC && vi.kp <= kMaxKBlocks * kKBlock) ? 1u : 0u;
    pd.eps_abs = pair_eps(vi, vj, w.e0);
    {
      uint32_t nchunks = vi.n_pad / kChunk, bits = 4;
      while ((1u << bits) < nchunks) ++bits;
      pd.chunk_bits = bits;
    }
    all.push_back(bp);
  }
  if (all.empty()) return R3D_OK;
  if (want_matches && (flags & R3D_MATCH_NO_COORD_DEDUP) == 0) {
    // per-view tables of the descent-free coordinate de-duplication (match_post.cpp), built once per upload
    std::vector<ViewDev*> need;
    for (auto& kv : w.views)
      if (kv.second.has_xy && !kv.second.ranks_tried) need.push_back(&kv.second);
    parallel_for(ctx->host_threads, need.size(), [&](size_t k) {
      ViewDev& v = *need[k];
      build_view_ranks(v.h_xy.data(), v.n, v.h_yrank, v.h_xshared, &v.n_slots);
      v.ranks_tried = true;
    });
  }
  const double t_prepared = now_ms();

  r3d_match_timing& T = w.timing;
  std::mutex t_mutex;  // T is updated by the batch tail threads

  // ---- output slots (double buffered) ------------------------------------------------------
  for (int sl = 0; sl < 2; ++sl) {
    OutSlot& o = w.out[sl];
    if (!o.d_counters) {
      R3D_CUDA_TRY(ctx, cudaMalloc(&o.d_counters, kCounterWords * sizeof(uint32_t)));
      R3D_CUDA_TRY(ctx, cudaMallocHost(&o.h_counters, kCounterWords * sizeof(uint32_t)));
      // blocking-sync events: the batch tails SLEEP in cudaEventSynchronize instead of spinning -- with two or three
      // batches in flight the default (spin) burned 2-3 CPUs per rank, a quarter of a 12-CPU-per-GPU container quota
      for (auto& e : o.ev) R3D_CUDA_TRY(ctx, cudaEventCreateWithFlags(&e, cudaEventBlockingSync));
    }
  }

  // ---- batches ---------------------------------------------------------------------------------
  // Batches bound the scratch memory and let the device->host copy, the bucketing and the host
  // de-duplication of batch b overlap the device work of batch b+1 (the reference's
  // order-dependent std::set step stays on the host).  Kernels of consecutive batches are stream
  // ordered; only the OUTPUT buffers (matches, counters) are double buffered.
  static const uint32_t kBatchPairs = []() {
    const char* e = getenv("R3D_BATCH_PAIRS");
    const int v = e ? atoi(e) : 0;
    return (uint32_t)std::min<int>(v > 0 ? v : 128, (int)kCounterWords - 16);
  }();
  const uint64_t kMaxRowsPerBatch = 24ull << 20;  // 24 Mi query rows -> 768 MiB of keys
  std::vector<std::thread> tails;
  std::shared_future<void> slot_free[2];
  std::atomic<int> tail_rc{R3D_OK};
  struct Joiner {
    std::vector<std::thread>& t;
    ~Joiner() { for (auto& x : t) if (x.joinable()) x.join(); }
  } joiner{tails};

  // candidate work items: 256 query rows on the integer path (four consumer warpgroups share each database tile),
  // 128 on the fp16 path
  const uint32_t qrows = item_rows(dtype, dim);
  size_t b0 = 0;
  uint32_t batch_no = 0;
  while (b0 < all.size()) {
    size_t b1 = b0;
    uint64_t rows = 0, qtotal = 0, n_items = 0;
    uint32_t max_nJ = 0, max_chunks = 0, max_nI = 0;
    // batches shrink geometrically towards the end so that the un-overlapped tail (copy + host
    // de-duplication of the LAST batch) is short
    const size_t remaining = all.size() - b0;
    const size_t this_batch = std::min<size_t>(kBatchPairs, std::max<size_t>(24, remaining / 2));
    while (b1 < all.size() && (b1 - b0) < this_batch && (rows + all[b1].pd.nJ_pad <= kMaxRowsPerBatch || b1 == b0)) {
      all[b1].pd.q_ofs = (uint32_t)rows;
      rows += all[b1].pd.nJ_pad;
      qtotal += all[b1].pd.nJ;
      if (all[b1].pd.use_tc) {
        n_items += all[b1].pd.nJ_pad / qrows;
        max_chunks = std::max(max_chunks, all[b1].pd.nI_pad / (uint32_t)kChunk);
      }
      max_nJ = std::max(max_nJ, all[b1].pd.nJ);
      max_nI = std::max(max_nI, all[b1].pd.nI);
      ++b1;
    }
    const uint32_t nb = (uint32_t)(b1 - b0);
    const uint32_t cstride = max_chunks + 1;
    auto hp = std::make_shared<std::vector<PairDesc>>(nb);
    for (uint32_t k = 0; k < nb; ++k) (*hp)[k] = all[b0 + k].pd;
    auto hitems = std::make_shared<std::vector<WorkItem>>();
    hitems->reserve(n_items + nb);
    for (uint32_t k = 0; k < nb; ++k)
      if ((*hp)[k].use_tc)
        for (uint32_t qb = 0; qb < (*hp)[k].nJ_pad / qrows; ++qb) hitems->push_back(WorkItem{k, qb});
    const bool any_tc = !hitems->empty();
    if (cascade)  // the item array carries (table row of I, table row of J) per pair instead of work items
      for (uint32_t k = 0; k < nb; ++k)
        hitems->push_back(WorkItem{w.views.find((*hp)[k].I)->second.cascade_index, w.views.find((*hp)[k].J)->second.cascade_index});

    const int sl = (int)(batch_no & 1u);
    OutSlot& o = w.out[sl];
    if (slot_free[sl].valid()) slot_free[sl].wait();  // batch b-2 has left this slot's buffers
    if (tail_rc.load() != R3D_OK) break;

    if ((rc = ensure_capacity<PairDesc>(ctx, &w.d_pairs, &w.pairs_cap, nb))) return rc;
    if ((rc = ensure_capacity<WorkItem>(ctx, &w.d_items, &w.items_cap, std::max<size_t>(hitems->size(), 1)))) return rc;
    if ((rc = ensure_capacity<uint4>(ctx, &w.d_keys, &w.keys_cap, rows * (kKeyStride / 4)))) return rc;
    if ((rc = ensure_capacity<uint2>(ctx, &w.d_fb, &w.fb_cap, qtotal))) return rc;
    if (any_tc) {
      if ((rc = ensure_capacity<uint32_t>(ctx, &w.d_cnt, &w.cnt_cap, (size_t)nb * cstride))) return rc;
      if ((rc = ensure_capacity<uint32_t>(ctx, &w.d_slot, &w.slot_cap, rows * 2))) return rc;
      if ((rc = ensure_capacity<uint32_t>(ctx, &w.d_list, &w.list_cap, rows * 2))) return rc;
      if ((rc = ensure_capacity<uint4>(ctx, &w.d_parts, &w.parts_cap, rows * 2))) return rc;
      if ((rc = ensure_capacity<uint2>(ctx, &w.d_list2, &w.list2_cap, qtotal))) return rc;
    }
    if (want_matches) {
      if ((rc = ensure_capacity<uint2>(ctx, &o.d_matches, &o.matches_cap, qtotal))) return rc;
      if ((rc = ensure_capacity<uint2>(ctx, &w.d_mdense, &w.mdense_cap, rows))) return rc;
    } else {
      if ((rc = ensure_capacity<float4>(ctx, &w.d_nn, &w.nn_cap, rows))) return rc;
    }
    // (re)allocations above are synchronous w.r.t. the device: previously enqueued work is done
    {  // uploads out of the slot's pinned staging buffer: truly asynchronous, the GPU keeps two batches queued
      const size_t pb = (size_t)nb * sizeof(PairDesc), ib = hitems->size() * sizeof(WorkItem);
      if (o.h_stage_cap < pb + ib) {
        if (o.h_stage) cudaFreeHost(o.h_stage);
        o.h_stage = nullptr;
        o.h_stage_cap = 0;
        R3D_CUDA_TRY(ctx, cudaMallocHost(&o.h_stage, (pb + ib) * 2));
        o.h_stage_cap = (pb + ib) * 2;
      }
      std::memcpy(o.h_stage, hp->data(), pb);
      std::memcpy((char*)o.h_stage + pb, hitems->data(), ib);
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(w.d_pairs, o.h_stage, pb, cudaMemcpyHostToDevice, w.stream));
      if (ib) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(w.d_items, (char*)o.h_stage + pb, ib, cudaMemcpyHostToDevice, w.stream));
    }
    R3D_CUDA_TRY(ctx, cudaMemsetAsync(o.d_counters, 0, (16 + nb) * sizeof(uint32_t), w.stream));
    uint64_t launches = 0;

    uint2* d_matches = want_matches ? (uint2*)w.d_mdense : nullptr;  // per-pair segments; packed into o.d_matches below
    float4* d_nn = want_matches ? nullptr : (float4*)w.d_nn;

    R3D_CUDA_TRY(ctx, cudaEventRecord(o.ev[0], w.stream));
    if (any_tc) {
      rc = launch_l2_candidates(ctx, w, (const PairDesc*)w.d_pairs, (const WorkItem*)w.d_items, (uint32_t)hitems->size(),
                                (uint32_t*)w.d_keys, dtype, dim);
      if (rc) return rc;
      launches += 1;
    }
    R3D_CUDA_TRY(ctx, cudaEventRecord(o.ev[1], w.stream));
    if (keys_dbg) {
      keys_dbg->resize(rows * (kKeyStride / 4));
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(keys_dbg->data(), w.d_keys, rows * (kKeyStride / 4) * sizeof(uint4), cudaMemcpyDeviceToHost, w.stream));
      R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    }
    if (any_tc) {
      if ((rc = launch_rerank_binned(ctx, w, (const PairDesc*)w.d_pairs, nb, max_nJ, cstride, (const uint32_t*)w.d_keys,
                                     dim, dtype, ratio2, (uint32_t*)w.d_cnt, (uint32_t*)w.d_slot, (uint32_t*)w.d_list,
                                     w.d_parts, o.d_counters, d_matches, (uint2*)w.d_list2, (uint2*)w.d_fb, d_nn))) return rc;
      if ((rc = launch_rerank_list(ctx, w, (const PairDesc*)w.d_pairs, (const uint32_t*)w.d_keys, w.d_parts, (const uint2*)w.d_list2,
                                   &o.d_counters[4], (uint32_t)std::min<uint64_t>(qtotal, 0xffffffffu), dim, dtype, ratio2,
                                   o.d_counters, d_matches, (uint2*)w.d_fb, d_nn))) return rc;
      launches += 6;
    }
    R3D_CUDA_TRY(ctx, cudaEventRecord(o.ev[2], w.stream));
    bool any_exact = false;
    for (uint32_t k = 0; k < nb; ++k) any_exact |= ((*hp)[k].use_tc == 0);
    if (cascade) {
      any_exact = false;
      if ((rc = launch_cascade_match(ctx, w, (const PairDesc*)w.d_pairs, (const uint2*)w.d_items, nb, max_nJ, max_nI, dim, dtype, ratio2,
                                     o.d_counters, d_matches))) return rc;
      launches += 1;
    }
    if (any_exact) {
      if ((rc = launch_fill_all_queries(ctx, w, (const PairDesc*)w.d_pairs, nb, (uint2*)w.d_fb, &o.d_counters[1]))) return rc;
      launches += 1;
    }
    if (!cascade) {
      if ((rc = launch_exact_scan(ctx, w, (const PairDesc*)w.d_pairs, (const uint2*)w.d_fb, &o.d_counters[1],
                                  (uint32_t)std::min<uint64_t>(qtotal, 0xffffffffu), dim, dtype, ratio2, o.d_counters,
                                  d_matches, d_nn))) return rc;
      launches += 1;
    }
    if (want_matches) {
      if ((rc = launch_pack_matches(ctx, w, (const PairDesc*)w.d_pairs, nb, o.d_counters + 16, (const uint2*)w.d_mdense,
                                    (uint2*)o.d_matches))) return rc;
      launches += 1;
    }
    R3D_CUDA_TRY(ctx, cudaEventRecord(o.ev[3], w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(o.h_counters, o.d_counters, (16 + nb) * sizeof(uint32_t), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaEventRecord(o.ev[4], w.stream));

    if (!want_matches) {  // r3d_search_neighbours / diagnostics: synchronous, single batch
      nn_out->resize(rows);
      R3D_CUDA_TRY(ctx, cudaMemcpyAsync(nn_out->data(), w.d_nn, rows * sizeof(float4), cudaMemcpyDeviceToHost, w.stream));
      R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
      T.d2h_bytes += rows * sizeof(float4);
      T.kernel_launches += launches;
      T.queries += qtotal;
      T.fallback_queries += o.h_counters[1];
      b0 = b1;
      ++batch_no;
      continue;
    }

    // ---- tail of the batch on its own host thread -------------------------------------------
    auto copied = std::make_shared<std::promise<void>>();
    slot_free[sl] = copied->get_future().share();
    const size_t base = b0;
    const bool cd = (flags & R3D_MATCH_NO_COORD_DEDUP) == 0;
    const int nthreads = std::max(1, ctx->host_threads / 2);
    const uint64_t h2d_batch = nb * sizeof(PairDesc) + hitems->size() * sizeof(WorkItem);
    tails.emplace_back([&, hp, hitems, copied, sl, nb, base, cd, nthreads, qtotal, launches, h2d_batch]() {
      OutSlot& os = w.out[sl];
      bool released = false;
      auto release = [&]() { if (!released) { released = true; copied->set_value(); } };
      auto bail = [&](const char* what, cudaError_t e) {
        tail_rc.store(fail(ctx, R3D_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e)));
        release();
      };
      cudaError_t e = cudaSetDevice(w.device);
      if (e != cudaSuccess) return bail("cudaSetDevice", e);
      e = cudaEventSynchronize(os.ev[4]);
      if (e != cudaSuccess) return bail("batch kernels", e);
      float ms_c = 0, ms_r = 0, ms_f = 0, ms_t = 0;
      cudaEventElapsedTime(&ms_c, os.ev[0], os.ev[1]);
      cudaEventElapsedTime(&ms_r, os.ev[1], os.ev[2]);
      cudaEventElapsedTime(&ms_f, os.ev[2], os.ev[3]);
      cudaEventElapsedTime(&ms_t, os.ev[0], os.ev[3]);
      // the matches arrive bucketed by pair: cnt = prefix sums of the per-pair counters
      std::vector<uint32_t> cnt(nb + 1, 0u);
      for (uint32_t k = 0; k < nb; ++k) cnt[k + 1] = cnt[k] + os.h_counters[16 + k];
      const uint32_t n_matches = cnt[nb];
      const uint32_t c_fb = os.h_counters[1], c_b = os.h_counters[4], c_c = os.h_counters[3], c_rej = os.h_counters[5];
      size_t bytes = (size_t)n_matches * sizeof(uint2);
      if (n_matches) {
        if (os.h_matches_cap < bytes) {
          if (os.h_matches) cudaFreeHost(os.h_matches);
          os.h_matches = nullptr;
          os.h_matches_cap = 0;
          e = cudaMallocHost(&os.h_matches, bytes + bytes / 2);
          if (e != cudaSuccess) return bail("cudaMallocHost", e);
          os.h_matches_cap = bytes + bytes / 2;
        }
        e = cudaMemcpyAsync(os.h_matches, os.d_matches, bytes, cudaMemcpyDeviceToHost, w.copy_stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(w.copy_stream);
        if (e != cudaSuccess) return bail("match copy", e);
      }
      const double t0 = now_ms();
      // out of the pinned buffer (uint2 (i, j) == r3d_indmatch) into the batch's result slab, so that the slot can
      // be handed to batch b+2; the pairs are de-duplicated in place and the result spans point into the slab
      r3d_indmatch* bucket = nullptr;
      r3d_slab slab = acquire_slab(n_matches, &bucket);  // recycled storage: no mmap / page faults in steady state
      if (n_matches) std::memcpy(bucket, os.h_matches, bytes);
      release();  // the slot's device + pinned buffers may be reused by batch b+2
      {
        std::lock_guard<std::mutex> lk(slab_mutex);
        slabs.push_back(slab);
      }
      const size_t n_groups = ((size_t)nb + kPostLanes - 1) / kPostLanes;
      parallel_for(nthreads, n_groups, [&](size_t g) {  // kPostLanes pairs per work item, advanced in lockstep
        r3d_indmatch* seg[kPostLanes];
        size_t n[kPostLanes];
        const float* xi[kPostLanes];
        const float* xj[kPostLanes];
        ViewRankRef rk[kPostLanes];
        uint32_t idx[kPostLanes];
        int lanes = 0;
        for (size_t k = g * kPostLanes; k < std::min<size_t>((g + 1) * kPostLanes, nb); ++k) {
          if (cnt[k + 1] == cnt[k]) continue;
          const ViewDev& vi = w.views.find((*hp)[k].I)->second;
          const ViewDev& vj = w.views.find((*hp)[k].J)->second;
          seg[lanes] = bucket + cnt[k];
          n[lanes] = cnt[k + 1] - cnt[k];
          xi[lanes] = vi.has_xy ? vi.h_xy.data() : nullptr;
          xj[lanes] = vj.has_xy ? vj.h_xy.data() : nullptr;
          rk[lanes] = (vi.has_xy && vi.n > 0 && vi.h_yrank.size() == vi.n) ? ViewRankRef{vi.h_yrank.data(), vi.h_xshared.data(), vi.n_slots}
                                                                : ViewRankRef{nullptr, nullptr, 0};
          idx[lanes] = (uint32_t)k;
          ++lanes;
        }
        if (!lanes) return;
        static const bool classic = getenv("R3D_DEDUP_CLASSIC") != nullptr;  // A/B: lockstep classic replay
        post_process_pairs(lanes, seg, n, xi, xj, cd, classic ? nullptr : rk);
        for (int t = 0; t < lanes; ++t) results[all[base + idx[t]].src_index] = r3d_span{seg[t], n[t]};
      });
      const double host_ms = now_ms() - t0;
      std::lock_guard<std::mutex> lk(t_mutex);
      T.ms_candidates += ms_c; T.ms_rerank += ms_r; T.ms_fallback += ms_f; T.ms_device_total += ms_t;
      T.ms_host_post += host_ms;
      T.kernel_launches += launches;
      T.queries += qtotal;
      T.fallback_queries += c_fb;
      T.third_chunk_queries += c_b;
      T.fifth_chunk_queries += c_c;
      T.rejected_queries += c_rej;
      T.d2h_bytes += (16 + nb) * sizeof(uint32_t) + bytes;
      T.h2d_bytes += h2d_batch;
    });
    b0 = b1;
    ++batch_no;
  }
  const double t_launch_done = now_ms();
  for (auto& t : tails) t.join();
  tails.clear();
  if (getenv("R3D_DEBUG_TIMING"))
    fprintf(stderr, "[r3d] match_on_worker: prepare %.2f ms, launch loop %.2f ms, tail join %.2f ms\n",
            t_prepared - t_enter, t_launch_done - t_prepared, now_ms() - t_launch_done);
  if (tail_rc.load() != R3D_OK) return tail_rc.load();
  return R3D_OK;
}

}  // namespace r3d

using namespace r3d;

extern "C" {

static int match_pairs_impl(r3d_ctx* ctx, const uint32_t* pairs, uint64_t n_pairs, float dist_ratio, uint32_t flags,
                            r3d_matches** out);

int r3d_match_pairs(r3d_ctx* ctx, const uint32_t* pairs, uint64_t n_pairs, float dist_ratio, uint32_t flags,
                    r3d_matches** out) {
  if (!ctx || !out || (n_pairs && !pairs)) return fail(ctx, R3D_ERR_INVALID, "r3d_match_pairs: bad arguments");
  *out = nullptr;
  if (!(flags & R3D_MATCH_MUTUAL_NN)) return match_pairs_impl(ctx, pairs, n_pairs, dist_ratio, flags, out);
  if (flags & R3D_MATCH_CASCADE_HASHING)
    return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_match_pairs: the mutual-NN select is defined for the exact matcher only");
  // Optional mutual-nearest-neighbour select (north_star; NOT part of the reference's MatchDistanceRatio, SURVEY.md A.2):
  // a match (i in I, j in J) of the forward pass survives iff j is also the nearest neighbour of i among J's
  // descriptors.  Second pass = the same matcher on the swapped pairs with the ratio test disabled.
  r3d_matches* fwd = nullptr;
  int rc = match_pairs_impl(ctx, pairs, n_pairs, dist_ratio, flags & ~R3D_MATCH_MUTUAL_NN, &fwd);
  if (rc) return rc;
  const r3d_match_timing t_fwd = ctx->match_timing;
  std::vector<uint32_t> rev_pairs(2 * n_pairs);
  for (uint64_t p = 0; p < n_pairs; ++p) { rev_pairs[2 * p] = pairs[2 * p + 1]; rev_pairs[2 * p + 1] = pairs[2 * p]; }
  r3d_matches* rev = nullptr;
  rc = match_pairs_impl(ctx, rev_pairs.data(), n_pairs, 1e18f, (flags & R3D_MATCH_EXACT_SCAN) | R3D_MATCH_NO_COORD_DEDUP, &rev);
  if (rc) { r3d_free_matches(fwd); return rc; }
  std::map<std::pair<uint32_t, uint32_t>, uint64_t> rev_of;
  for (uint64_t k = 0; k < rev->pairs.size() / 2; ++k) rev_of[{rev->pairs[2 * k], rev->pairs[2 * k + 1]}] = k;
  r3d_matches* m = new r3d_matches();
  std::vector<uint32_t> nn_in_J;
  for (uint64_t k = 0; k < fwd->pairs.size() / 2; ++k) {
    const uint32_t I = fwd->pairs[2 * k], J = fwd->pairs[2 * k + 1];
    auto it = rev_of.find({J, I});
    if (it == rev_of.end()) continue;
    // rev entry (i_ = feature of J, j_ = feature of I): the nearest neighbour in J of I's feature j_
    const r3d_span& rs = rev->per[it->second];
    uint32_t maxi = 0;
    for (const r3d_indmatch& e : rs) maxi = std::max(maxi, e.j);
    nn_in_J.assign((size_t)maxi + 1, 0xffffffffu);
    for (const r3d_indmatch& e : rs) nn_in_J[e.j] = e.i;
    std::vector<r3d_indmatch> keep;
    for (const r3d_indmatch& e : fwd->per[k])
      if (e.i <= maxi && nn_in_J[e.i] == e.j) keep.push_back(e);
    if (!keep.empty()) m->push(I, J, std::move(keep));
  }
  r3d_free_matches(fwd);
  r3d_free_matches(rev);
  {  // both passes count
    r3d_match_timing& t = ctx->match_timing;
    t.ms_candidates += t_fwd.ms_candidates; t.ms_rerank += t_fwd.ms_rerank; t.ms_fallback += t_fwd.ms_fallback;
    t.ms_device_total += t_fwd.ms_device_total; t.ms_host_post += t_fwd.ms_host_post; t.kernel_launches += t_fwd.kernel_launches;
    t.queries += t_fwd.queries; t.fallback_queries += t_fwd.fallback_queries; t.rejected_queries += t_fwd.rejected_queries;
    t.h2d_bytes += t_fwd.h2d_bytes; t.d2h_bytes += t_fwd.d2h_bytes;
  }
  *out = m;
  return R3D_OK;
}

static int match_pairs_impl(r3d_ctx* ctx, const uint32_t* pairs, uint64_t n_pairs, float dist_ratio, uint32_t flags,
                            r3d_matches** out) {
  *out = nullptr;
  const double t_call = now_ms();
  const uint64_t h2d_uploads = ctx->pending_h2d;  // uploads since the previous call belong to this one
  ctx->pending_h2d = 0;
  for (auto& wk : ctx->workers) wk.timing = r3d_match_timing{};
  const size_t nw = ctx->workers.size();
  if (nw == 0) return fail(ctx, R3D_ERR_INVALID, "r3d_match_pairs: context has no device");
  if (flags & R3D_MATCH_CASCADE_HASHING) {
    // the hash tables depend on the zero-mean descriptor of ALL views of the matching job: without an explicit
    // r3d_cascade_prepare() that covers this pair list, the job is this call (the reference's behaviour)
    bool ready = true;
    for (auto& wk : ctx->workers) ready = ready && cascade_ready(wk, pairs, n_pairs);
    if (!ready) {
      std::set<uint32_t> su(pairs, pairs + 2 * n_pairs);
      const std::vector<uint32_t> used(su.begin(), su.end());
      for (auto& wk : ctx->workers) {
        const int rc = cascade_prepare(ctx, wk, used);
        if (rc) return rc;
      }
    }
  }
  // Shard the (I-sorted) pair list into contiguous, cost-balanced ranges: one per device, no
  // collective; every device holds all regions.
  DeviceWorker& w0 = ctx->workers[0];
  const std::vector<uint64_t> cut = balanced_cuts(n_pairs, nw, [&](uint64_t p) {
    auto a = w0.views.find(pairs[2 * p]), b = w0.views.find(pairs[2 * p + 1]);
    return (a != w0.views.end() && b != w0.views.end()) ? (double)a->second.n * (double)b->second.n : 0.0;
  });
  std::vector<std::vector<r3d_span>> res(nw);
  std::vector<std::vector<r3d_slab>> res_slabs(nw);
  const int rc = fan_out(ctx, [&](size_t k, DeviceWorker& w) {
    return match_on_worker(ctx, w, pairs + 2 * cut[k], cut[k + 1] - cut[k], dist_ratio, flags, res[k], res_slabs[k], nullptr);
  });
  if (rc) return rc;
  {
    r3d_match_timing sum{};
    for (auto& wk : ctx->workers) {
      const r3d_match_timing& t = wk.timing;
      sum.ms_candidates = std::max(sum.ms_candidates, t.ms_candidates);
      sum.ms_rerank = std::max(sum.ms_rerank, t.ms_rerank);
      sum.ms_fallback = std::max(sum.ms_fallback, t.ms_fallback);
      sum.ms_device_total = std::max(sum.ms_device_total, t.ms_device_total);
      sum.ms_host_post = std::max(sum.ms_host_post, t.ms_host_post);
      sum.kernel_launches += t.kernel_launches;
      sum.queries += t.queries;
      sum.fallback_queries += t.fallback_queries;
      sum.third_chunk_queries += t.third_chunk_queries;
      sum.fifth_chunk_queries += t.fifth_chunk_queries;
      sum.rejected_queries += t.rejected_queries;
      sum.h2d_bytes += t.h2d_bytes;
      sum.d2h_bytes += t.d2h_bytes;
    }
    sum.h2d_bytes += h2d_uploads;
    ctx->match_timing = sum;
  }
  // assemble the PairWiseMatches map (sorted by (I,J); empty pairs are not inserted)
  const double t_assemble = now_ms();
  struct Entry { uint32_t I, J; r3d_span* v; };
  std::vector<Entry> entries;
  for (size_t k = 0; k < nw; ++k)
    for (uint64_t p = 0; p < res[k].size(); ++p)
      if (!res[k][p].empty()) entries.push_back(Entry{pairs[2 * (cut[k] + p)], pairs[2 * (cut[k] + p) + 1], &res[k][p]});
  std::stable_sort(entries.begin(), entries.end(), [](const Entry& a, const Entry& b) {
    return a.I < b.I || (a.I == b.I && a.J < b.J);
  });
  r3d_matches* m = new r3d_matches();
  m->pairs.reserve(2 * entries.size());
  m->per.reserve(entries.size());
  for (size_t e = 0; e < entries.size(); ++e) {
    if (e > 0 && entries[e].I == entries[e - 1].I && entries[e].J == entries[e - 1].J) continue;  // map::insert keeps the first
    m->push_span(entries[e].I, entries[e].J, *entries[e].v);
  }
  for (auto& sl : res_slabs) m->slabs.insert(m->slabs.end(), sl.begin(), sl.end());
  if (getenv("R3D_DEBUG_TIMING"))
    fprintf(stderr, "[r3d] r3d_match_pairs total %.2f ms (assembly %.2f ms)\n", now_ms() - t_call, now_ms() - t_assemble);
  *out = m;
  return R3D_OK;
}

int r3d_search_neighbours(r3d_ctx* ctx, uint32_t view_db, uint32_t view_query, int32_t* idx, float* dist) {
  if (!ctx || !idx || !dist) return fail(ctx, R3D_ERR_INVALID, "r3d_search_neighbours: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  auto iI = w.views.find(view_db), iJ = w.views.find(view_query);
  if (iI == w.views.end() || iJ == w.views.end()) return fail(ctx, R3D_ERR_INVALID, "r3d_search_neighbours: unknown view");
  if (iI->second.n < 2 || iJ->second.n < 1)
    return fail(ctx, R3D_ERR_INVALID, "r3d_search_neighbours: NN > number of database rows (upstream returns false)");
  const uint32_t pr[2] = {view_db, view_query};
  std::vector<r3d_span> dummy;
  std::vector<r3d_slab> dummy_slabs;
  std::vector<float4> nn;
  if (iI->second.dim != iJ->second.dim || iI->second.dtype != iJ->second.dtype)
    return fail(ctx, R3D_ERR_INVALID, "r3d_search_neighbours: descriptor type mismatch");
  w.timing = r3d_match_timing{};
  int rc = match_on_worker(ctx, w, pr, 1, 1.0f, R3D_MATCH_DEFAULT, dummy, dummy_slabs, &nn);
  if (rc) return rc;
  ctx->match_timing = w.timing;
  const uint32_t nq = iJ->second.n;
  if (nn.size() < nq) return fail(ctx, R3D_ERR_INVALID, "r3d_search_neighbours: no result");
  for (uint32_t q = 0; q < nq; ++q) {
    uint32_t i1, i2;
    std::memcpy(&i1, &nn[q].x, 4);
    std::memcpy(&i2, &nn[q].y, 4);
    idx[2 * q] = (int32_t)i1;
    idx[2 * q + 1] = (int32_t)i2;
    dist[2 * q] = nn[q].z;
    dist[2 * q + 1] = nn[q].w;
  }
  return R3D_OK;
}

int r3d_debug_candidate_keys(r3d_ctx* ctx, uint32_t view_db, uint32_t view_query, uint32_t* keys, float* eps_abs) {
  // keys: n_query_pad x 8 uint32 (6 keys + 2 unused)
  if (!ctx || !keys) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_candidate_keys: bad arguments");
  DeviceWorker& w = ctx->workers[0];
  auto iI = w.views.find(view_db), iJ = w.views.find(view_query);
  if (iI == w.views.end() || iJ == w.views.end()) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_candidate_keys: unknown view");
  const uint32_t pr[2] = {view_db, view_query};
  std::vector<r3d_span> dummy;
  std::vector<r3d_slab> dummy_slabs;
  std::vector<float4> nn;
  std::vector<uint4> k;
  int rc = match_on_worker(ctx, w, pr, 1, 1.0f, R3D_MATCH_DEFAULT, dummy, dummy_slabs, &nn, &k);
  if (rc) return rc;
  std::memcpy(keys, k.data(), k.size() * sizeof(uint4));
  if (eps_abs) *eps_abs = pair_eps(iI->second, iJ->second, w.e0);
  return R3D_OK;
}

}  // extern "C"
