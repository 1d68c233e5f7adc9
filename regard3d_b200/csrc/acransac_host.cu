// acransac_host.cu -- host side of AC-RANSAC: the F / H / E filters (r3d_filter_pairs; r3d_relative_poses runs the
// essential one), the driver of the persistent kernel that the filters and r3d_resect_views share, and the
// log-combinatorial tables.
//
// Replaces ImageCollectionGeometricFilter::Robust_model_estimation(GeometricFilter_FMatrix_AC(4.0,
// 2048), putatives, false) + Get_geometric_matches() (src/R3DComputeMatches.cpp:2099-2115).
//
// ACRANSAC (SURVEY.md A.5) is sequential per pair, so one CTA of k_acransac_fused (acransac_fused.cu) runs a pair from
// its first sample to its final inlier list.  The sample stream is drawn on the device by a restatement of
// std::mt19937 + std::uniform_int_distribution (acransac_rng.cuh); rng_selftest() checks it against this process's
// <random>, and every AC-RANSAC entry point returns R3D_ERR_UNSUPPORTED when the two disagree.  The host builds each
// pair's adaptor (normalisation, logalpha0, loge0), ships the putative (i, j) lists through pinned staging, launches
// the set-up kernels and one persistent launch per size class, and after ONE synchronisation copies the inlier lists
// back through the same staging.
#include "acransac.cuh"
#include "acransac_rng.cuh"
#include "detmath.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace r3d {

// log-combinatorial tables (float, upstream makelogcombi_n / makelogcombi_k).  logcombi(k,n) is a running float sum over
// i = 1..min(k,n-k): its partial sums ARE the entries for smaller k, so one O(n) pass reproduces the upstream O(n^2)
// table bit for bit.
int AcTables::upload(r3d_ctx* ctx, DeviceWorker& w, uint32_t ns, uint32_t maxM, uint64_t tbl_total) {
  h_vlog10.resize(maxM + 2);
  for (uint32_t k = 0; k <= maxM + 1; ++k) h_vlog10[k] = std::log10((float)k);
  h_logc_k.assign(maxM + 1, 0.f);
  for (uint32_t n = 0; n <= maxM; ++n) {
    uint32_t k = ns;
    if (k >= n) continue;
    if (n - k < k) k = n - k;
    float r = 0.f;
    for (uint32_t i = 1; i <= k; ++i) r += h_vlog10[n - i + 1] - h_vlog10[i];
    h_logc_k[n] = r;
  }
  if (!vlog10.alloc(h_vlog10.size()) || !logc_n.alloc(tbl_total) || !logc_k.alloc(h_logc_k.size()))
    return fail(ctx, R3D_ERR_NOMEM, "AC-RANSAC tables: device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(vlog10.p, h_vlog10.data(), h_vlog10.size() * sizeof(float), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(logc_k.p, h_logc_k.data(), h_logc_k.size() * sizeof(float), cudaMemcpyHostToDevice, w.stream));
  return R3D_OK;
}

int AcFused::plan(r3d_ctx* ctx, DeviceWorker& w, int model_, const std::vector<AcPair>& pairs) {
  // the persistent kernel draws the sample stream on the device; it needs the restated std::uniform_int_distribution to
  // agree with this process's <random> (acransac_rng.cuh)
  if (!rng_selftest())
    return fail(ctx, R3D_ERR_UNSUPPORTED, "AC-RANSAC: the device sample stream disagrees with this process's <random>");
  model = model_;
  const uint32_t n = (uint32_t)pairs.size();
  std::vector<uint32_t> cls[kClasses];
  uint32_t huge_maxM = 0;
  for (uint32_t a = 0; a < n; ++a) {
    const uint32_t M = pairs[a].M;
    int c = 0;
    while (c < 5 && (1024u << c) < M) ++c;
    if (M > 16384u) { c = 5; huge_maxM = std::max(huge_maxM, M); }
    cls[c].push_back(a);
  }
  // the scratch is shared by the class launches (same stream): sized for the largest grid x cap
  size_t si_need = 0, huge_need = 0;
  horder.clear();
  for (int c = 0; c < kClasses; ++c) {
    std::stable_sort(cls[c].begin(), cls[c].end(), [&](uint32_t x, uint32_t y) { return pairs[x].M > pairs[y].M; });
    class_ofs[c] = (uint32_t)horder.size();
    horder.insert(horder.end(), cls[c].begin(), cls[c].end());
    const uint32_t cnt = (uint32_t)cls[c].size();
    if (!cnt) continue;
    const bool huge = c == 5;
    uint32_t cap = 1024u << c;
    if (huge) {
      cap = 32768;
      while (cap < huge_maxM) cap <<= 1;
    }
    uint32_t grid = std::min<uint32_t>(cnt, (uint32_t)w.sm_count * (uint32_t)acransac_fused_ctas_per_sm(model, cap, huge));
    if (huge) grid = std::min<uint32_t>(grid, (uint32_t)w.sm_count);
    caps[c] = cap;
    grids[c] = grid;
    si_need = std::max(si_need, (size_t)grid * cap);
    if (huge) huge_need = (size_t)grid * cap;
  }
  class_ofs[kClasses] = n;
  if (!order.alloc(n) || !work.alloc(kClasses) || !si.alloc(si_need) || !se.alloc(huge_need) || !pool.alloc(huge_need))
    return fail(ctx, R3D_ERR_NOMEM, "AC-RANSAC: device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(order.p, horder.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(work.p, 0, kClasses * sizeof(uint32_t), w.stream));
  return R3D_OK;
}

int AcFused::launch(r3d_ctx* ctx, DeviceWorker& w, const AcPair* d_pairs, const double2* x1, const double2* x2, const double* x3,
                    const float* logc_n, const float* logc_k, uint32_t max_iter, const uint2* matches, uint2* out_matches,
                    AcFusedOut* out, double* out_model, uint64_t& launches) {
  for (int c = kClasses - 1; c >= 0; --c) {  // the long-running classes first
    const uint32_t cnt = class_ofs[c + 1] - class_ofs[c];
    if (!cnt) continue;
    const int rc = launch_acransac_fused(ctx, w, model, c == 5, d_pairs, order.p + class_ofs[c], cnt, work.p + c, x1, x2, logc_n,
                                         logc_k, caps[c], max_iter, se.p, si.p, pool.p, matches, out_matches, out, out_model,
                                         grids[c], x3);
    if (rc) return rc;
    launches += 1;
  }
  return R3D_OK;
}

namespace {

// the worker's two pinned buffers that stage the filters' (i, j) lists, to the device and back
constexpr size_t kStageElems = (size_t)4 << 20;  // 32 MB of (i, j) per buffer
int ensure_fstage(r3d_ctx* ctx, DeviceWorker& w) {
  if (w.h_fstage_cap >= kStageElems) return R3D_OK;
  for (void*& hp : w.h_fstage) {
    if (hp) cudaFreeHost(hp);
    hp = nullptr;
    R3D_CUDA_TRY(ctx, cudaMallocHost(&hp, kStageElems * sizeof(uint2)));
  }
  w.h_fstage_cap = kStageElems;
  return R3D_OK;
}

struct Chunk { uint32_t a0, a1; size_t lo, hi; };  // pairs [a0, a1), their (i, j) lists [lo, hi)
// the pairs (laid out in pt_ofs order, a ascending) in chunks that fit a staging buffer; a single pair larger than
// that is a chunk of its own
std::vector<Chunk> stage_chunks(const std::vector<AcPair>& hpairs) {
  const uint32_t n = (uint32_t)hpairs.size();
  std::vector<Chunk> chunks;
  uint32_t a = 0;
  while (a < n) {
    Chunk c{a, a, hpairs[a].pt_ofs, hpairs[a].pt_ofs};
    while (c.a1 < n && ((size_t)hpairs[c.a1].pt_ofs + hpairs[c.a1].M - c.lo <= kStageElems || c.a1 == c.a0)) {
      c.hi = (size_t)hpairs[c.a1].pt_ofs + hpairs[c.a1].M;
      ++c.a1;
    }
    chunks.push_back(c);
    a = c.a1;
  }
  return chunks;
}

// The AC-RANSAC of the filter's pairs (size classes, one persistent launch per class, largest pairs first); ONE
// synchronisation, then the inlier lists come back through pinned staging.
int run_fused(r3d_ctx* ctx, DeviceWorker& w, int model, uint32_t max_iter, const std::vector<uint32_t>& src,
              const std::vector<AcPair>& hpairs, const AcPair* d_pairs, const double2* d_x1, const double2* d_x2,
              const uint2* d_match, const AcTables& tab, uint32_t pt_total, uint32_t sizeSample, double t_begin,
              r3d_filter_timing& T, std::vector<std::vector<r3d_indmatch>>& result, std::vector<AcBestModel>* best) {
  const uint32_t n = (uint32_t)hpairs.size();
  AcFused fused(w);
  int rc = fused.plan(ctx, w, model, hpairs);
  if (rc) return rc;
  DevArr<AcFusedOut> d_out(w);
  DevArr<uint2> d_outm(w);
  DevArr<double> d_model(w);
  if (!d_out.alloc(n) || !d_outm.alloc(pt_total) || (best && !d_model.alloc((size_t)n * 9)))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_filter_pairs: device scratch");
  Events<2> ev;
  R3D_CUDA_TRY(ctx, ev.create());
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[0], w.stream));
  rc = fused.launch(ctx, w, d_pairs, d_x1, d_x2, nullptr, tab.logc_n.p, tab.logc_k.p, max_iter, d_match, d_outm.p, d_out.p,
                    best ? d_model.p : nullptr, T.kernel_launches);
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaEventRecord(ev.e[1], w.stream));
  std::vector<AcFusedOut> hout(n);
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hout.data(), d_out.p, (size_t)n * sizeof(AcFusedOut), cudaMemcpyDeviceToHost, w.stream));
  std::vector<double> hmodel(best ? (size_t)n * 9 : 0);
  if (best)
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hmodel.data(), d_model.p, hmodel.size() * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  if (best)
    for (uint32_t a = 0; a < n; ++a) {
      const AcFusedOut& o = hout[a];
      if (!(o.minNFA < 0) || !((double)o.n_inliers > sizeSample * 2.5)) continue;
      AcBestModel& b = (*best)[src[a]];
      std::memcpy(b.model, &hmodel[9 * (size_t)a], sizeof(b.model));
      b.errorMax = o.errorMax;
    }
  const float ms = ev.ms(0, 1);
  T.ms_score = ms;
  T.ms_solve = 0.0;
  T.rounds = 1;
  for (const AcFusedOut& o : hout) T.hypotheses += o.iterations;
  if (getenv("R3D_DEBUG_TIMING")) {
    uint64_t ex = 0, mo = 0, evs = 0;
    for (const AcFusedOut& o : hout) { ex += o.exact_scores; mo += o.models; evs += o.events; }
    fprintf(stderr, "[r3d] fused filter: %u pairs, kernel %.2f ms, %llu iterations, %llu models, %llu exact (%.2f %%), %llu events\n", n, ms,
            (unsigned long long)T.hypotheses, (unsigned long long)mo, (unsigned long long)ex, 100.0 * (double)ex / (double)std::max<uint64_t>(mo, 1),
            (unsigned long long)evs);
  }
  const double t_after_kernel = now_ms();
  // ---- inlier lists back: chunks of whole pairs through two pinned staging buffers, copied out by the host pool ----
  // GeometricFilter_*Matrix_AC::Robust_estimation keeps the pair iff #inliers > MINIMUM_SAMPLES * 2.5
  rc = ensure_fstage(ctx, w);
  if (rc) return rc;
  const std::vector<Chunk> chunks = stage_chunks(hpairs);
  std::vector<uint2> big;  // a single pair larger than the staging buffer
  Events<2> cev;
  R3D_CUDA_TRY(ctx, cev.create(false));
  auto issue = [&](size_t ci) -> cudaError_t {
    const Chunk& c = chunks[ci];
    if (c.hi - c.lo > kStageElems) return cudaSuccess;  // handled synchronously below
    // only the inlier prefix of each pair is meaningful, but one contiguous copy beats thousands of small ones
    cudaError_t e = cudaMemcpyAsync(w.h_fstage[ci & 1], d_outm.p + c.lo, (c.hi - c.lo) * sizeof(uint2), cudaMemcpyDeviceToHost, w.stream);
    if (e != cudaSuccess) return e;
    return cudaEventRecord(cev.e[ci & 1], w.stream);
  };
  if (!chunks.empty()) R3D_CUDA_TRY(ctx, issue(0));
  for (size_t ci = 0; ci < chunks.size(); ++ci) {
    const Chunk& c = chunks[ci];
    const uint2* base;
    if (c.hi - c.lo > kStageElems) {
      big.resize(c.hi - c.lo);
      R3D_CUDA_TRY(ctx, cudaMemcpy(big.data(), d_outm.p + c.lo, (c.hi - c.lo) * sizeof(uint2), cudaMemcpyDeviceToHost));
      base = big.data();
    } else {
      R3D_CUDA_TRY(ctx, cudaEventSynchronize(cev.e[ci & 1]));
      base = (const uint2*)w.h_fstage[ci & 1];
    }
    if (ci + 1 < chunks.size()) R3D_CUDA_TRY(ctx, issue(ci + 1));  // the other buffer: free since chunk ci - 1 was consumed
    parallel_for(ctx->host_threads, c.a1 - c.a0, [&](size_t k) {
      const uint32_t a = c.a0 + (uint32_t)k;
      const AcFusedOut& o = hout[a];
      if (!(o.minNFA < 0) || !((double)o.n_inliers > sizeSample * 2.5)) return;
      const r3d_indmatch* sp = (const r3d_indmatch*)(base + (hpairs[a].pt_ofs - c.lo));
      result[src[a]].assign(sp, sp + o.n_inliers);
    });
  }
  if (getenv("R3D_DEBUG_TIMING"))
    fprintf(stderr, "[r3d] fused filter total %.2f ms (kernel %.2f, results back %.2f)\n", now_ms() - t_begin, T.ms_score, now_ms() - t_after_kernel);
  T.ms_device_total = T.ms_score;
  T.ms_host = now_ms() - t_begin - T.ms_device_total;
  return R3D_OK;
}


}  // namespace

// pairs [p0, p1) of the putative map on worker w; result (sized by the caller to the whole map) is indexed by pair
int filter_pairs_model(r3d_ctx* ctx, DeviceWorker& w, int model, double precision_px, uint32_t max_iter, const r3d_matches* put,
                   const r3d_view_info* views, uint32_t n_views, uint64_t p0, uint64_t p1, r3d_filter_timing& T,
                   std::vector<std::vector<r3d_indmatch>>& result, std::vector<AcBestModel>* best) {
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  T = r3d_filter_timing{};
  const double t_begin = now_ms();
  const uint32_t sizeSample = ac_min_samples(model), MAX_MODELS = ac_max_models(model);  // Kernel::MINIMUM_SAMPLES / MAX_MODELS

  // ---- per pair set-up (kernel adaptor of SURVEY.md A.5: normalisation, logalpha0, tables) ----
  std::vector<uint32_t> src;   // index of every pair in the putative map
  std::vector<AcPair> hpairs;
  uint64_t pt_total = 0, tbl_total = 0;  // (i, j) of every putative match / logc_n entries, pair after pair
  uint32_t maxM = 0;
  for (uint64_t p = p0; p < p1; ++p) {
    const uint32_t I = put->pairs[2 * p], J = put->pairs[2 * p + 1];
    const uint32_t M = (uint32_t)put->per[p].size();
    if (M <= sizeSample) continue;  // ACRANSAC returns at once: nData <= MINIMUM_SAMPLES
    if (I >= n_views || J >= n_views) return fail(ctx, R3D_ERR_INVALID, "r3d_filter_pairs: view id outside views[]");
    // GeometricFilter_EMatrix_AC::Robust_estimation returns false without two valid pinhole intrinsics
    if (model == 2 && (!(views[I].focal > 0.0) || !(views[J].focal > 0.0))) continue;
    auto vi = w.views.find(I), vj = w.views.find(J);
    if (vi == w.views.end() || vj == w.views.end() || !vi->second.has_xy || !vj->second.has_xy)
      return fail(ctx, R3D_ERR_INVALID, "r3d_filter_pairs: positions of a view were not uploaded");
    AcPair ap;
    std::memset(&ap, 0, sizeof(ap));
    ap.pt_ofs = (uint32_t)pt_total; ap.M = M; ap.tbl_ofs = (uint32_t)tbl_total;
    src.push_back((uint32_t)p);
    hpairs.push_back(ap);
    pt_total += M;
    tbl_total += M + 2;  // logc_n[0..M] and the table's error bound (k_ac_tables)
    maxM = std::max(maxM, M);
  }
  if (src.empty()) return R3D_OK;
  if (pt_total > 0xfffffff0ull) return fail(ctx, R3D_ERR_UNSUPPORTED, "r3d_filter_pairs: too many putative matches in one call");
  const uint32_t n = (uint32_t)src.size();
  std::vector<AcPointSrc> hsrc(n);
  const double t_pairs0 = now_ms();
  parallel_for(ctx->host_threads, n, [&](size_t a) {
    const uint32_t I = put->pairs[2 * (size_t)src[a]], J = put->pairs[2 * (size_t)src[a] + 1];
    const uint32_t M = hpairs[a].M;
    const ViewDev& vi = w.views.find(I)->second;
    const ViewDev& vj = w.views.find(J)->second;
    const int wI = (int)views[I].width, hI = (int)views[I].height, wJ = (int)views[J].width, hJ = (int)views[J].height;
    // the essential adaptor keeps pixel coordinates (normalizer = identity)
    const double s1 = model == 2 ? 1.0 : 1.0 / std::sqrt((double)(wI * hI));
    const double s2 = model == 2 ? 1.0 : 1.0 / std::sqrt((double)(wJ * hJ));
    const double c1x = model == 2 ? 0.0 : (double)(-.5f * wI) * s1, c1y = model == 2 ? 0.0 : -.5 * hI * s1;
    const double c2x = model == 2 ? 0.0 : (double)(-.5f * wJ) * s2, c2y = model == 2 ? 0.0 : -.5 * hJ * s2;
    // the matched positions are looked up, promoted to double and normalised on the device (k_ac_points):
    // the host only ships the (i, j) list
    static_assert(sizeof(r3d_indmatch) == sizeof(uint2), "IndMatch layout");
    AcPointSrc& ps = hsrc[a];
    ps.xyI = vi.d_xy; ps.xyJ = vj.d_xy;
    ps.s1 = s1; ps.c1x = c1x; ps.c1y = c1y; ps.s2 = s2; ps.c2x = c2x; ps.c2y = c2y;
    ps.nI = vi.n; ps.nJ = vj.n; ps.identity = model == 2 ? 1u : 0u; ps.pad_ = 0;
    AcPair& ap = hpairs[a];
    const double precision = precision_px * precision_px;  // upper_bound_precision = Square(dPrecision)
    ap.max_thr = precision * s2 * s2;
    if (model == 0) {  // point-to-line
      const double D = std::sqrt((double)wJ * (double)wJ + (double)hJ * (double)hJ);
      const double Aarea = (double)wJ * (double)hJ;
      ap.logalpha0 = dm::log10_det(2.0 * D / Aarea / s2);
    } else if (model == 2) {  // ACKernelAdaptorEssential: log10(2 D / A * .5), pixel units
      const double D = std::sqrt((double)wJ * (double)wJ + (double)hJ * (double)hJ);
      const double Aarea = (double)wJ * (double)hJ;
      ap.logalpha0 = dm::log10_det(2.0 * D / Aarea * .5);
    } else {           // point-to-point
      ap.logalpha0 = dm::log10_det(R3D_PI / ((double)wJ * (double)hJ) / (s2 * s2));
    }
    ap.loge0 = dm::log10_det((double)MAX_MODELS * (double)(M - sizeSample));
    ap.K[0] = views[I].focal; ap.K[1] = views[I].ppx; ap.K[2] = views[I].ppy;
    ap.K[3] = views[J].focal; ap.K[4] = views[J].ppx; ap.K[5] = views[J].ppy;
  });
  if (getenv("R3D_DEBUG_TIMING"))
    fprintf(stderr, "[r3d] filter set-up: pair scan %.2f ms, per-pair adaptors %.2f ms\n", t_pairs0 - t_begin, now_ms() - t_pairs0);

  // ---- device buffers -------------------------------------------------------------------------
  DevArr<AcPair> d_pairs(w);
  DevArr<AcPointSrc> d_src(w);
  DevArr<double2> d_x1(w), d_x2(w);
  DevArr<uint2> d_match(w);
  DevArr<uint32_t> d_bad(w);
  if (!d_pairs.alloc(n) || !d_src.alloc(n) || !d_x1.alloc(pt_total) || !d_x2.alloc(pt_total) || !d_match.alloc(pt_total) ||
      !d_bad.alloc(1))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_filter_pairs: device scratch");
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_pairs.p, hpairs.data(), n * sizeof(AcPair), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_src.p, hsrc.data(), n * sizeof(AcPointSrc), cudaMemcpyHostToDevice, w.stream));
  // the putative (i, j) lists: gathered by the host pool into two pinned staging buffers, chunk by chunk, while the
  // previous chunk is on its way to the device (a pageable 800 MB source at C3 would move at a fraction of the link)
  {
    int rc = ensure_fstage(ctx, w);
    if (rc) return rc;
    Events<2> uev;
    R3D_CUDA_TRY(ctx, uev.create(false));
    size_t chunk_no = 0;
    for (const Chunk& c : stage_chunks(hpairs)) {
      if (c.hi - c.lo > kStageElems) {  // one pair larger than the staging buffer: straight from its (pageable) span
        R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_match.p + c.lo, put->per[src[c.a0]].data(), (c.hi - c.lo) * sizeof(uint2), cudaMemcpyHostToDevice, w.stream));
        R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
      } else {
        const int buf = (int)(chunk_no & 1);
        if (chunk_no >= 2) R3D_CUDA_TRY(ctx, cudaEventSynchronize(uev.e[buf]));  // the copy that last read this buffer is done
        uint2* stage = (uint2*)w.h_fstage[buf];
        parallel_for(ctx->host_threads, c.a1 - c.a0, [&](size_t k) {
          const size_t a = c.a0 + k;
          std::memcpy(stage + (hpairs[a].pt_ofs - c.lo), put->per[src[a]].data(), (size_t)hpairs[a].M * sizeof(uint2));
        });
        R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_match.p + c.lo, stage, (c.hi - c.lo) * sizeof(uint2), cudaMemcpyHostToDevice, w.stream));
        R3D_CUDA_TRY(ctx, cudaEventRecord(uev.e[buf], w.stream));
        ++chunk_no;
      }
    }
  }
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(d_bad.p, 0, sizeof(uint32_t), w.stream));
  {
    int rcp = launch_ac_points(ctx, w, d_pairs.p, d_src.p, n, d_match.p, d_x1.p, d_x2.p, d_bad.p);
    if (rcp) return rcp;
    uint32_t hbad = 0;
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(&hbad, d_bad.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
    if (hbad) return fail(ctx, R3D_ERR_INVALID, "r3d_filter_pairs: match index out of range");
    T.kernel_launches += 1;
  }
  // logc_n tables: float prefix sums over the host's log10 table, one thread per pair in the upstream order
  AcTables tab(w);
  int rc = tab.upload(ctx, w, sizeSample, maxM, tbl_total);
  if (rc) return rc;
  rc = launch_ac_tables(ctx, w, d_pairs.p, n, tab.vlog10.p, tab.logc_n.p);
  if (rc) return rc;
  T.kernel_launches += 1;
  if (getenv("R3D_DEBUG_TIMING")) fprintf(stderr, "[r3d] filter host set-up + point upload: %.2f ms\n", now_ms() - t_begin);
  return run_fused(ctx, w, model, max_iter, src, hpairs, d_pairs.p, d_x1.p, d_x2.p, d_match.p, tab, (uint32_t)pt_total, sizeSample,
                   t_begin, T, result, best);
}

}  // namespace r3d

using namespace r3d;

// Diagnostics (host only): 1 when the device-side restatement of std::mt19937 + std::uniform_int_distribution
// (acransac_rng.cuh) reproduces this process's <random>; without it the AC-RANSAC entry points return R3D_ERR_UNSUPPORTED.
extern "C" int r3d_debug_rng_selftest(void) { return rng_selftest() ? 1 : 0; }

extern "C" int r3d_debug_acransac_score(r3d_ctx* ctx, int model, uint32_t M, const double* x1, const double* x2, const double* x3,
                                        double max_thr, double logalpha0, const double* K, const double* models, uint32_t n_models,
                                        r3d_ac_score* out, double* lo, double* hi, double* e, float* logc_n, float* logc_k) {
  if (!ctx || model < 0 || model > 3 || !x1 || !x2 || !K || !models || !out || n_models < 1)
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: bad arguments");
  const uint32_t NS = ac_min_samples(model), MS = ac_model_size(model);
  if ((model == 3) != (x3 != nullptr)) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: x3 belongs to model 3");
  if (M < NS || M > (1u << 24)) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: M outside [minimal sample, 2^24]");
  if (!(max_thr >= 0.0) || (model != 3 && !(max_thr < INFINITY)) || !std::isfinite(logalpha0))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: bad max_thr / logalpha0");
  if (model == 3 && !(K[3] > 0.0 && K[3] < INFINITY)) return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: K[3] must be > 0");
  if ((lo != nullptr) != (hi != nullptr) || (lo != nullptr) != (e != nullptr))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: lo, hi and e go together");
  if (n_models > (1u << 20) || (lo && (uint64_t)n_models * M > (1ull << 28)))
    return fail(ctx, R3D_ERR_INVALID, "r3d_debug_acransac_score: too many models");
  DeviceWorker& w = ctx->workers[0];
  R3D_CUDA_TRY(ctx, cudaSetDevice(w.device));
  AcPair ap;
  std::memset(&ap, 0, sizeof(ap));
  ap.M = M;
  ap.max_thr = max_thr;
  ap.logalpha0 = logalpha0;
  ap.loge0 = dm::log10_det((double)ac_max_models(model) * (double)(M - NS));
  std::memcpy(ap.K, K, sizeof(ap.K));
  std::vector<double2> h1(M), h2(M);
  for (uint32_t i = 0; i < M; ++i) {
    h1[i] = make_double2(x1[2 * i], x1[2 * i + 1]);
    h2[i] = make_double2(x2[2 * i], x2[2 * i + 1]);
  }
  const uint32_t cap = debug_acransac_cap(M);
  const size_t nper = lo ? (size_t)n_models * M : 0;
  DevArr<AcPair> d_pair(w);
  DevArr<double2> d_x1(w), d_x2(w);
  DevArr<double> d_x3(w), d_models(w), d_se(w), d_lo(w), d_hi(w), d_e(w);
  DevArr<uint32_t> d_si(w);
  DevArr<r3d_ac_score> d_out(w);
  AcTables tab(w);
  if (!d_pair.alloc(1) || !d_x1.alloc(M) || !d_x2.alloc(M) || !d_x3.alloc(M) || !d_models.alloc((size_t)n_models * MS) ||
      !d_se.alloc(cap) || !d_si.alloc(cap) || !d_out.alloc(n_models) ||
      (nper && (!d_lo.alloc(nper) || !d_hi.alloc(nper) || !d_e.alloc(nper))))
    return fail(ctx, R3D_ERR_NOMEM, "r3d_debug_acransac_score: device scratch");
  int rc = tab.upload(ctx, w, NS, M, (uint64_t)M + 2);
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_pair.p, &ap, sizeof(ap), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_x1.p, h1.data(), (size_t)M * sizeof(double2), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_x2.p, h2.data(), (size_t)M * sizeof(double2), cudaMemcpyHostToDevice, w.stream));
  if (x3) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_x3.p, x3, (size_t)M * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(d_models.p, models, (size_t)n_models * MS * sizeof(double), cudaMemcpyHostToDevice, w.stream));
  rc = launch_ac_tables(ctx, w, d_pair.p, 1, tab.vlog10.p, tab.logc_n.p);
  if (rc) return rc;
  rc = debug_acransac_score(ctx, w, model, d_pair.p, d_x1.p, d_x2.p, x3 ? d_x3.p : nullptr, tab.logc_n.p, tab.logc_k.p, d_models.p,
                            n_models, M, d_se.p, d_si.p, d_out.p, nper ? d_lo.p : nullptr, nper ? d_hi.p : nullptr,
                            nper ? d_e.p : nullptr);
  if (rc) return rc;
  R3D_CUDA_TRY(ctx, cudaMemcpyAsync(out, d_out.p, (size_t)n_models * sizeof(r3d_ac_score), cudaMemcpyDeviceToHost, w.stream));
  if (nper) {
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(lo, d_lo.p, nper * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(hi, d_hi.p, nper * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
    R3D_CUDA_TRY(ctx, cudaMemcpyAsync(e, d_e.p, nper * sizeof(double), cudaMemcpyDeviceToHost, w.stream));
  }
  if (logc_n) R3D_CUDA_TRY(ctx, cudaMemcpyAsync(logc_n, tab.logc_n.p, ((size_t)M + 2) * sizeof(float), cudaMemcpyDeviceToHost, w.stream));
  R3D_CUDA_TRY(ctx, cudaStreamSynchronize(w.stream));
  if (logc_k) std::memcpy(logc_k, tab.h_logc_k.data(), tab.h_logc_k.size() * sizeof(float));
  return R3D_OK;
}

extern "C" int r3d_filter_pairs(r3d_ctx* ctx, int model, double precision_px, uint32_t max_iter, const r3d_matches* putative,
                                const r3d_view_info* views, uint32_t n_views, r3d_matches** out) {
  if (!ctx || !putative || !views || !out) return fail(ctx, R3D_ERR_INVALID, "r3d_filter_pairs: bad arguments");
  *out = nullptr;
  if (model != R3D_MODEL_F && model != R3D_MODEL_H && model != R3D_MODEL_E)
    return fail(ctx, R3D_ERR_INVALID, "r3d_filter_pairs: unknown model");
  const int internal = model == R3D_MODEL_F ? 0 : (model == R3D_MODEL_H ? 1 : 2);
  const uint64_t P_all = putative->pairs.size() / 2;
  std::vector<std::vector<r3d_indmatch>> res(P_all);
  // image pairs are independent: cut the map into contiguous ranges of equal putative-match counts, one per device
  // of the context (every device holds all positions), no collective -- the same rule as r3d_match_pairs
  const std::vector<uint64_t> cut = balanced_cuts(P_all, ctx->workers.size(), [&](uint64_t p) { return putative->per[p].size(); });
  std::vector<r3d_filter_timing> tms(ctx->workers.size());
  const int rc = fan_out(ctx, [&](size_t k, DeviceWorker& w) {
    return filter_pairs_model(ctx, w, internal, precision_px, max_iter, putative, views, n_views, cut[k], cut[k + 1], tms[k], res);
  });
  if (rc) return rc;
  {
    r3d_filter_timing sum{};
    for (const r3d_filter_timing& t : tms) {
      sum.ms_solve = std::max(sum.ms_solve, t.ms_solve);
      sum.ms_score = std::max(sum.ms_score, t.ms_score);
      sum.ms_device_total = std::max(sum.ms_device_total, t.ms_device_total);
      sum.ms_host = std::max(sum.ms_host, t.ms_host);
      sum.kernel_launches += t.kernel_launches;
      sum.hypotheses += t.hypotheses;
      sum.rounds = std::max(sum.rounds, t.rounds);
    }
    ctx->filter_timing = sum;
  }
  r3d_matches* m = new r3d_matches();
  const uint64_t P = putative->pairs.size() / 2;
  for (uint64_t p = 0; p < P; ++p) {
    if (res[p].empty()) continue;  // pairs whose estimation failed disappear from the map
    m->push(putative->pairs[2 * p], putative->pairs[2 * p + 1], std::move(res[p]));
  }
  *out = m;
  return R3D_OK;
}
