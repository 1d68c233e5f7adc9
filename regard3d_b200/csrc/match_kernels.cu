// match_kernels.cu -- CUDA-core kernels of the putative-matching path (sm_90a):
//   k_view_stats / k_view_prepare : build the fp16 tensor-core operands of a view (+ error constants; the exact
//                                   norms of the integer path)
//   k_rerank                      : exact re-rank of the candidate chunks, certification, ratio test
//   k_exact_scan                  : exact brute-force 2-NN for listed queries (uncertified / forced)
//
// "Exact" means: squared L2 accumulated in float in the order of openMVG::matching::L2<T>
// (4-way unrolled; the metric the reference names at src/R3DComputeMatches.cpp:290-291), using
// __fsub_rn/__fmul_rn/__fadd_rn so no FMA contraction can change a bit.
#include "r3d_internal.cuh"
#include "match_device.cuh"

namespace r3d {

// ------------------------------------------------------------------------------------------------
// k_rerank : one warp per listed (pair, query) -- stage B of the certification.  The query arrives
// with the exact top-2 of its two best chunks (stage A, rerank_binned.cu); the warp re-ranks the next
// kStageBChunks chunks (one lane per database row) and certifies against the key after them.
// ------------------------------------------------------------------------------------------------
constexpr int kStageBChunks = (32 / kChunk) < 3 ? (32 / kChunk) : 3;
struct PartB { float d1, d2; uint32_t i1, i2; };

template <int DTYPE>
__global__ void __launch_bounds__(256) k_rerank(const PairDesc* __restrict__ pairs,
                                                const uint32_t* __restrict__ keys, const PartB* __restrict__ parts,
                                                const uint2* __restrict__ list, const uint32_t* __restrict__ list_count,
                                                uint32_t dim, float ratio2, uint32_t* counters, uint2* matches,
                                                uint2* fallback, float4* nn) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_list = *list_count;
  for (uint32_t item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < n_list;
       item += gridDim.x * (blockDim.x >> 5)) {
    const uint2 pq = list[item];
    const uint32_t pair = pq.x, q = pq.y;
    const PairDesc pd = pairs[pair];
    const uint4 ka = __ldg((const uint4*)keys + (size_t)(pd.q_ofs + q) * (kKeyStride / 4));
    const uint4 kb = __ldg((const uint4*)keys + (size_t)(pd.q_ofs + q) * (kKeyStride / 4) + 1);
    const uint32_t key[6] = {ka.x, ka.y, ka.z, ka.w, kb.x, kb.y};
    const uint32_t nchunks = pd.nI_pad / kChunk;
    const uint32_t cmask = (1u << pd.chunk_bits) - 1u;
    const double pack_rel = ldexp(1.0, (int)pd.chunk_bits - 23);
    const size_t rb = row_bytes(DTYPE, dim);
    const char* qrow = (const char*)pd.descJ + (size_t)q * rb;
    const double gamma = (double)(dim + 16) * (1.0 / 16777216.0);
    const PartB pa = parts[(size_t)(pd.q_ofs + q) * 2 + 0];
    const PartB pb = parts[(size_t)(pd.q_ofs + q) * 2 + 1];
    Top2 t, tb;
    t.d1 = pa.d1; t.d2 = pa.d2; t.i1 = pa.i1; t.i2 = pa.i2;
    tb.d1 = pb.d1; tb.d2 = pb.d2; tb.i1 = pb.i1; tb.i2 = pb.i2;
    t = top2_merge(t, tb);
    Top2 u;
    u.d1 = u.d2 = FLT_MAX; u.i1 = u.i2 = 0xffffffffu;
    const uint32_t slot = lane / kChunk;  // which of the stage-B chunks this lane works on
    if (slot < (uint32_t)kStageBChunks) {
      const uint32_t c = key[2 + slot] & cmask;
      const uint32_t col = c * kChunk + (lane % kChunk);
      if (c < nchunks && col < pd.nI) {
        u.d1 = exact_l2<DTYPE>(qrow, (const char*)pd.descI + (size_t)col * rb, dim);
        u.i1 = col;
      }
    }
    u = top2_warp_reduce(u);
    t = top2_merge(t, u);
    const bool ok = key_lower_bound(key[2 + kStageBChunks], pd.eps_abs, gamma, pack_rel) > (double)t.d2;
    if (lane == 0) {
      if (ok) {
        emit_result(pd, pair, q, t, ratio2, counters, matches, nn);
      } else {
        const uint32_t s2 = atomicAdd(&counters[1], 1u);
        fallback[s2] = make_uint2(pair, q);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// k_exact_scan : exact brute force for the listed (pair, query) items.
//   long lists (whole pairs that bypass the tensor-core pass): one block per item;
//   short lists (the handful of uncertified queries per batch): every item is cut into kScanSlices row
//   slices handled by different blocks -- a 10 000-row scan by ONE block is a 0.3 ms latency chain per
//   launch -- the last slice to finish (per-item arrival counter) merges the partial top-2s and emits.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kScanSlices = 32;
constexpr uint32_t kScanSplitMaxItems = 2048;
template <int DTYPE>
__global__ void __launch_bounds__(256) k_exact_scan(const PairDesc* __restrict__ pairs,
                                                    const uint2* __restrict__ list,
                                                    const uint32_t* __restrict__ list_count, uint32_t dim,
                                                    float ratio2, uint32_t* counters, uint2* matches,
                                                    float4* nn, Top2* __restrict__ slice_best,
                                                    uint32_t* __restrict__ slice_done) {
  extern __shared__ __align__(16) unsigned char smem_q[];
  __shared__ Top2 warp_best[8];
  __shared__ uint32_t s_last;
  const uint32_t n_list = *list_count;
  if (n_list <= kScanSplitMaxItems && slice_best != nullptr) {
    for (uint32_t vb = blockIdx.x; vb < n_list * kScanSlices; vb += gridDim.x) {
      const uint32_t item = vb / kScanSlices, slice = vb % kScanSlices;
      const uint2 pq = list[item];
      const PairDesc pd = pairs[pq.x];
      const size_t rb = row_bytes(DTYPE, dim);
      const char* qrow = (const char*)pd.descJ + (size_t)pq.y * rb;
      __syncthreads();
      for (uint32_t b = threadIdx.x; b < rb; b += blockDim.x) smem_q[b] = qrow[b];
      __syncthreads();
      const uint32_t per = (pd.nI + kScanSlices - 1) / kScanSlices;
      const uint32_t r0 = slice * per, r1 = min(pd.nI, r0 + per);
      Top2 t;
      t.d1 = t.d2 = FLT_MAX; t.i1 = t.i2 = 0xffffffffu;
      for (uint32_t i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
        const float dd = exact_l2<DTYPE>(smem_q, (const char*)pd.descI + (size_t)i * rb, dim);
        top2_insert(t, dd, i);
      }
      t = top2_warp_reduce(t);
      if ((threadIdx.x & 31u) == 0) warp_best[threadIdx.x >> 5] = t;
      __syncthreads();
      if (threadIdx.x < 32) {
        Top2 u;
        u.d1 = u.d2 = FLT_MAX; u.i1 = u.i2 = 0xffffffffu;
        if (threadIdx.x < (blockDim.x >> 5)) u = warp_best[threadIdx.x];
        u = top2_warp_reduce(u);
        if (threadIdx.x == 0) {
          slice_best[(size_t)item * kScanSlices + slice] = u;
          __threadfence();
          s_last = (atomicAdd(&slice_done[item], 1u) == kScanSlices - 1u) ? 1u : 0u;
        }
      }
      __syncthreads();
      if (s_last && threadIdx.x < 32) {  // every slice of the item has been published
        __threadfence();
        static_assert(sizeof(Top2) == sizeof(uint4) && kScanSlices == 32, "one slice per lane");
        const uint4 raw = __ldcg((const uint4*)slice_best + (size_t)item * kScanSlices + threadIdx.x);  // L2, not L1
        Top2 u;
        u.d1 = __uint_as_float(raw.x); u.d2 = __uint_as_float(raw.y); u.i1 = raw.z; u.i2 = raw.w;
        u = top2_warp_reduce(u);
        if (threadIdx.x == 0) emit_result(pd, pq.x, pq.y, u, ratio2, counters, matches, nn);
      }
    }
    return;
  }
  for (uint32_t item = blockIdx.x; item < n_list; item += gridDim.x) {
    const uint2 pq = list[item];
    const PairDesc pd = pairs[pq.x];
    const size_t rb = row_bytes(DTYPE, dim);
    const char* qrow = (const char*)pd.descJ + (size_t)pq.y * rb;
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < rb; b += blockDim.x) smem_q[b] = qrow[b];
    __syncthreads();
    Top2 t;
    t.d1 = t.d2 = FLT_MAX; t.i1 = t.i2 = 0xffffffffu;
    for (uint32_t i = threadIdx.x; i < pd.nI; i += blockDim.x) {
      const float d = exact_l2<DTYPE>(smem_q, (const char*)pd.descI + (size_t)i * rb, dim);
      top2_insert(t, d, i);
    }
    t = top2_warp_reduce(t);
    if ((threadIdx.x & 31u) == 0) warp_best[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x < 32) {
      Top2 u;
      u.d1 = u.d2 = FLT_MAX; u.i1 = u.i2 = 0xffffffffu;
      if (threadIdx.x < (blockDim.x >> 5)) u = warp_best[threadIdx.x];
      u = top2_warp_reduce(u);
      if (threadIdx.x == 0) emit_result(pd, pq.x, pq.y, u, ratio2, counters, matches, nn);
    }
  }
}

__global__ void k_fill_all_queries(const PairDesc* __restrict__ pairs, uint32_t n_pairs, uint2* list,
                                   uint32_t* list_count) {
  const uint32_t pair = blockIdx.y;
  if (pair >= n_pairs) return;
  const PairDesc pd = pairs[pair];
  if (pd.use_tc) return;
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < pd.nJ; q += gridDim.x * blockDim.x) {
    const uint32_t slot = atomicAdd(list_count, 1u);
    list[slot] = make_uint2(pair, q);
  }
}

// ------------------------------------------------------------------------------------------------
// operand preparation
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_desc(const void* base, int dtype, size_t idx) {
  return dtype == 0 ? ((const float*)base)[idx] : (float)((const uint8_t*)base)[idx];
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// stats[0] = max ||a||^2, [1] = max ||fp16(a)||^2, [2] = max ||a - fp16(a)||^2, [3] = max |a_k|
// norms (integer path only, rows [0, n_pad)): the exact ||a||^2, kPadNorm on padding rows
__global__ void k_view_stats(const void* __restrict__ desc, int dtype, uint32_t n, uint32_t n_pad, uint32_t dim,
                             float* stats, int32_t* __restrict__ norms) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) {
    if (norms && row < n_pad && lane == 0) norms[row] = kPadNorm;
    return;
  }
  double n2 = 0, h2 = 0, d2 = 0;
  float ma = 0.f;
  for (uint32_t k = lane; k < dim; k += 32) {
    const float a = load_desc(desc, dtype, (size_t)row * dim + k);
    const float h = __half2float(__float2half_rn(a));
    n2 += (double)a * (double)a;
    h2 += (double)h * (double)h;
    const double e = (double)a - (double)h;
    d2 += e * e;
    ma = fmaxf(ma, fabsf(a));
  }
  n2 = warp_sum(n2); h2 = warp_sum(h2); d2 = warp_sum(d2); ma = warp_max(ma);
  if (lane == 0) {
    if (norms) norms[row] = (int32_t)n2;  // a sum of integer squares below 2^53: exact
    // non-negative floats order like their bit patterns; round UP so the maxima stay upper bounds
    atomicMax((unsigned int*)&stats[0], __float_as_uint(__double2float_ru(n2)));
    atomicMax((unsigned int*)&stats[1], __float_as_uint(__double2float_ru(h2)));
    atomicMax((unsigned int*)&stats[2], __float_as_uint(__double2float_ru(d2)));
    atomicMax((unsigned int*)&stats[3], __float_as_uint(ma));
  }
}

// Writes both operand matrices of a view.  Row layout (kmain = pad16(dim); kp >= kmain + 16 halves,
// zero padded to the row alignment):
//   database role opD: [ a_0 .. a_{dim-1} 0.. | p0 p1 S0 S1 0 x12 ]      ||a||^2 ~= p0*S0 + p1*S1
//   query role    opQ: [ -2a_0 .. -2a_{dim-1} 0.. | S0 S1 p0 p1 0 x12 ]
// so that  opQ_row . opD_row' = ||a'||^2 + ||a||^2 - 2 a.a'   (the squared distance).
// Padding rows of the database role get p0 = 65504 (they lose against every real row).
__global__ void k_view_prepare(const void* __restrict__ desc, int dtype, uint32_t n, uint32_t n_pad,
                               uint32_t dim, uint32_t kp, uint32_t kmain, int e0,
                               __half* __restrict__ opQ, __half* __restrict__ opD) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n_pad) return;
  const float S0 = ldexpf(1.f, e0), S1 = ldexpf(1.f, e0 - 11);
  __half* q = opQ + (size_t)row * kp;
  __half* d = opD + (size_t)row * kp;
  if (row >= n) {
    for (uint32_t k = lane; k < kp; k += 32) {
      q[k] = __float2half_rn(0.f);
      float v = 0.f;
      if (k == kmain) v = 65504.f;
      if (k == kmain + 2) v = S0;
      if (k == kmain + 3) v = S1;
      d[k] = __float2half_rn(v);
    }
    return;
  }
  double n2 = 0;
  for (uint32_t k = lane; k < kmain; k += 32) {
    float a = 0.f;
    if (k < dim) a = load_desc(desc, dtype, (size_t)row * dim + k);
    const __half h = __float2half_rn(a);
    d[k] = h;
    q[k] = __float2half_rn(-2.f * __half2float(h));
    n2 += (double)a * (double)a;
  }
  n2 = warp_sum(n2);
  if (lane < kBiasCols) {
    const double dS0 = (double)S0, dS1 = (double)S1;
    const __half p0 = __double2half(n2 / dS0);
    const double r = n2 - (double)__half2float(p0) * dS0;
    const __half p1 = __double2half(r / dS1);
    const __half z = __float2half_rn(0.f);
    const __half hS0 = __float2half_rn(S0), hS1 = __float2half_rn(S1);
    __half dv = z, qv = z;
    if (lane == 0) { dv = p0; qv = hS0; }
    if (lane == 1) { dv = p1; qv = hS1; }
    if (lane == 2) { dv = hS0; qv = p0; }
    if (lane == 3) { dv = hS1; qv = p1; }
    d[kmain + lane] = dv;
    q[kmain + lane] = qv;
  }
  for (uint32_t k = kmain + kBiasCols + lane; k < kp; k += 32) {  // alignment padding of the row
    d[k] = __float2half_rn(0.f);
    q[k] = __float2half_rn(0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
int launch_view_stats(r3d_ctx* ctx, DeviceWorker& w, ViewDev& v) {
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(v.d_stats, 0, 4 * sizeof(float), w.stream));
  const uint32_t rows = v.int_ops ? v.n_pad : v.n;
  if (rows == 0) return R3D_OK;
  const int wpb = 8;
  k_view_stats<<<(rows + wpb - 1) / wpb, wpb * 32, 0, w.stream>>>(v.d_desc, (int)v.dtype, v.n, v.n_pad, v.dim, v.d_stats,
                                                                  v.d_norm);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_view_prepare(r3d_ctx* ctx, DeviceWorker& w, ViewDev& v, int e0) {
  const int wpb = 8;
  k_view_prepare<<<(v.n_pad + wpb - 1) / wpb, wpb * 32, 0, w.stream>>>(v.d_desc, (int)v.dtype, v.n, v.n_pad,
                                                                     v.dim, v.kp, (uint32_t)pad_up((int)(v.dim ? v.dim : 16), 16), e0, v.d_opQ, v.d_opD);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_rerank_list(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const uint32_t* d_keys, const void* d_parts,
                       const uint2* d_list, const uint32_t* d_list_count, uint32_t max_list, uint32_t dim, int dtype,
                       float ratio2, uint32_t* d_counters, uint2* d_matches, uint2* d_fallback, float4* d_nn) {
  if (max_list == 0) return R3D_OK;
  const int wpb = 8;
  uint32_t grid = (max_list + wpb - 1) / wpb;
  if (grid > (uint32_t)w.sm_count * 16u) grid = (uint32_t)w.sm_count * 16u;
  if (dtype == 0)
    k_rerank<0><<<grid, wpb * 32, 0, w.stream>>>(d_pairs, d_keys, (const PartB*)d_parts, d_list, d_list_count, dim, ratio2,
                                                 d_counters, d_matches, d_fallback, d_nn);
  else
    k_rerank<1><<<grid, wpb * 32, 0, w.stream>>>(d_pairs, d_keys, (const PartB*)d_parts, d_list, d_list_count, dim, ratio2,
                                                 d_counters, d_matches, d_fallback, d_nn);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

// ---- pack the per-pair match segments for the host copy ----------------------------------------------
// one block per pair: offset = sum of the counts of the pairs before it (<= a few thousand values), then the pair's
// segment goes to the packed array -- SORTED by (i, j) when it fits the shared-memory bitonic network
// (<= kPackSortCap matches): IndMatch::getDeduplicated wants that order, and the sort is microseconds here but a
// third of the host tail's CPU time.  Larger segments are copied as they are (the host checks the order and sorts
// when needed, so the order is a performance matter only).
constexpr uint32_t kPackSortCap = 8192;
__global__ void __launch_bounds__(256) k_pack_matches(const PairDesc* __restrict__ pairs, const uint32_t* __restrict__ pair_cnt,
                                                      const uint2* __restrict__ dense, uint2* __restrict__ packed) {
  extern __shared__ __align__(16) unsigned long long s_key[];  // kPackSortCap keys: i << 32 | j
  __shared__ uint32_t s_part[8];
  __shared__ uint32_t s_ofs;
  const uint32_t p = blockIdx.x;
  uint32_t acc = 0;
  for (uint32_t k = threadIdx.x; k < p; k += blockDim.x) acc += pair_cnt[k];
  for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31u) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < 8; ++w) t += s_part[w];
    s_ofs = t;
  }
  __syncthreads();
  const uint32_t n = pair_cnt[p], src = pairs[p].q_ofs, dst = s_ofs;
  if (n < 2 || n > kPackSortCap) {
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) packed[dst + k] = dense[src + k];
    return;
  }
  uint32_t P = 2;
  while (P < n) P <<= 1;
  for (uint32_t k = threadIdx.x; k < P; k += blockDim.x) {
    unsigned long long key = ~0ull;  // padding sorts last
    if (k < n) {
      const uint2 m = dense[src + k];
      key = ((unsigned long long)m.x << 32) | m.y;
    }
    s_key[k] = key;
  }
  __syncthreads();
  for (uint32_t size = 2; size <= P; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
        const uint32_t lo = (t / stride) * (stride << 1) + (t % stride);
        const uint32_t hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = s_key[lo], b = s_key[hi];
        if ((a > b) == up) { s_key[lo] = b; s_key[hi] = a; }
      }
      __syncthreads();
    }
  }
  for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
    const unsigned long long key = s_key[k];
    packed[dst + k] = make_uint2((uint32_t)(key >> 32), (uint32_t)key);
  }
}

int launch_pack_matches(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, uint32_t n_pairs, const uint32_t* d_pair_cnt,
                        const uint2* d_dense, uint2* d_packed) {
  if (!n_pairs) return R3D_OK;
  const size_t smem = (size_t)kPackSortCap * sizeof(unsigned long long);
  R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_pack_matches, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_pack_matches<<<n_pairs, 256, smem, w.stream>>>(d_pairs, d_pair_cnt, d_dense, d_packed);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_exact_scan(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const uint2* d_list,
                      const uint32_t* d_list_count, uint32_t max_list, uint32_t dim, int dtype, float ratio2,
                      uint32_t* d_counters, uint2* d_matches, float4* d_nn) {
  if (max_list == 0) return R3D_OK;
  // scratch of the split mode: partial top-2 per (item, slice) + per-item arrival counters (zeroed per launch)
  const size_t best_bytes = (size_t)kScanSplitMaxItems * kScanSlices * sizeof(Top2);
  const size_t need = best_bytes + (size_t)kScanSplitMaxItems * sizeof(uint32_t);
  int rc = ensure_capacity<unsigned char>(ctx, &w.d_scan, &w.scan_cap, need);
  if (rc) return rc;
  Top2* slice_best = (Top2*)w.d_scan;
  uint32_t* slice_done = (uint32_t*)((unsigned char*)w.d_scan + best_bytes);
  R3D_CUDA_TRY(ctx, cudaMemsetAsync(slice_done, 0, (size_t)kScanSplitMaxItems * sizeof(uint32_t), w.stream));
  const uint32_t want = max_list < kScanSplitMaxItems ? max_list * kScanSlices : max_list;
  const uint32_t grid = want < (uint32_t)(w.sm_count * 8) ? want : (uint32_t)(w.sm_count * 8);
  const size_t smem = (dtype == 0 ? (size_t)dim * 4 : (size_t)dim) + 16;
  if (dtype == 0)
    k_exact_scan<0><<<grid, 256, smem, w.stream>>>(d_pairs, d_list, d_list_count, dim, ratio2, d_counters, d_matches, d_nn,
                                                   slice_best, slice_done);
  else
    k_exact_scan<1><<<grid, 256, smem, w.stream>>>(d_pairs, d_list, d_list_count, dim, ratio2, d_counters, d_matches, d_nn,
                                                   slice_best, slice_done);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

int launch_fill_all_queries(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, uint32_t n_pairs,
                            uint2* d_list, uint32_t* d_list_count) {
  if (n_pairs == 0) return R3D_OK;
  dim3 grid(64, n_pairs);
  k_fill_all_queries<<<grid, 256, 0, w.stream>>>(d_pairs, n_pairs, d_list, d_list_count);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

}  // namespace r3d
