// k_l2_candidates.cu -- the tensor-core candidate kernel (sm_90a: TMA, mbarrier, wgmma).
//
// Work item = (pair, 128-query block of view J).  For every query row the kernel evaluates the fp16 distance
// surrogate opQ(J) . opD(I) against all database rows of view I and keeps the kNumKeys smallest chunk minima
// (kChunk consecutive database rows each), packed with the chunk id, in keys_out.
//
// Persistent CTAs (one per SM, 227 KB of shared memory), three warpgroups:
//   warpgroup 0      one TMA producer warp: the item's query block (nkb boxes of 128 rows x 64 columns, double
//                    buffered across items) and a ring of database stages (one 64-column K-block of a 256-row tile)
//   warpgroups 1, 2  consumers of query rows 0-63 / 64-127: per 256-row tile, m64n256k16 wgmma into 128 f32
//                    registers per thread, then the chunk minima and the key insertion in registers.
// Both consumers read every database stage.  The tensor core runs one consumer's tile while the other reduces its
// accumulator, so the epilogue overlaps the MMAs without a second accumulator.
// Barriers: full[s] (TMA bytes landed), empty[s] (the 8 consumer warps are done with the stage), qfull / qempty the
// same for the query buffers.
#include "r3d_internal.cuh"
#include "tc_ptx.cuh"

namespace r3d {

using namespace tcx;

namespace {

constexpr int kMaxStages = 8;
constexpr uint32_t kTileN = 256;                  // database rows per tile (the wgmma N extent)
constexpr uint32_t kStageBytes = 2 * kBoxBytes;   // one K-block of a 256-row tile: two 128-row TMA boxes
constexpr uint32_t kConsumerWarps = 8;
constexpr uint32_t kThreads = 384;
constexpr size_t kSmemOptIn = 232448;             // 227 KB: the largest dynamic shared memory of one block on sm_90
static_assert(kChunk == 8, "the epilogue reduces one 8-column block of the wgmma accumulator per chunk");

// Minima of four consecutive chunks of one accumulator row, spread over the 4 lanes of a quad (2 columns each),
// reduced and scattered so that lane q of the quad ends with the minimum of chunk q: 3 shuffles for 4 chunks.
__device__ __forceinline__ float quad_min4(float p0, float p1, float p2, float p3, uint32_t q) {
  const bool b1 = (q & 2u) != 0, b0 = (q & 1u) != 0;
  const float k0 = fminf(b1 ? p2 : p0, __shfl_xor_sync(0xffffffffu, b1 ? p0 : p2, 2));
  const float k1 = fminf(b1 ? p3 : p1, __shfl_xor_sync(0xffffffffu, b1 ? p1 : p3, 2));
  return fminf(b0 ? k1 : k0, __shfl_xor_sync(0xffffffffu, b0 ? k0 : k1, 1));
}

// the kNumKeys smallest keys of this lane's set and the set of lane ^ d (the keys of different chunks differ)
__device__ __forceinline__ void merge_keys(float (&key)[kNumKeys], int d) {
  float y[kNumKeys];
#pragma unroll
  for (int i = 0; i < kNumKeys; ++i) y[i] = __shfl_xor_sync(0xffffffffu, key[i], d);
#pragma unroll
  for (int i = 0; i < kNumKeys; ++i) {
    float x = y[i];
#pragma unroll
    for (int j = 0; j < kNumKeys - 1; ++j) {
      const float hi = fmaxf(key[j], x);
      key[j] = fminf(key[j], x);
      x = hi;
    }
    key[kNumKeys - 1] = fminf(key[kNumKeys - 1], x);
  }
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 1)
k_l2_candidates(const CUtensorMap* __restrict__ tmapQ, const CUtensorMap* __restrict__ tmapD,
                const PairDesc* __restrict__ pairs, const WorkItem* __restrict__ items, uint32_t n_items,
                uint32_t* __restrict__ keys_out, uint32_t nkb, uint32_t ksteps, uint32_t n_stages, uint32_t n_qbuf) {
  extern __shared__ unsigned char smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  // n_qbuf (1 or 2) x nkb boxes: the item's 128 query rows.  With two buffers the next item's query block is loaded
  // while the current item's last tiles are still in the tensor pipe.
  const uint32_t q_base = base;
  const uint32_t q_bytes = nkb * kBoxBytes;
  const uint32_t d_base = q_base + n_qbuf * q_bytes;            // n_stages stages
  const uint32_t bar_full = d_base + n_stages * kStageBytes;    // [kMaxStages]
  const uint32_t bar_empty = bar_full + 8 * kMaxStages;         // [kMaxStages]
  const uint32_t bar_qfull = bar_empty + 8 * kMaxStages;        // [2]
  const uint32_t bar_qempty = bar_qfull + 16;                   // [2]

  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < (uint32_t)kMaxStages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kConsumerWarps);
    }
    for (uint32_t qb = 0; qb < 2; ++qb) {
      mbar_init(bar_qfull + 8 * qb, 1);
      mbar_init(bar_qempty + 8 * qb, kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ========================================= TMA producer =========================================
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    uint32_t stage = 0, phase = 0, qi = 0;
    for (uint32_t it = blockIdx.x; it < n_items; it += gridDim.x, ++qi) {
      const WorkItem wi = items[it];
      const PairDesc pd = pairs[wi.pair];
      const CUtensorMap* mq = tmapQ + pd.slotJ;
      const CUtensorMap* md = tmapD + pd.slotI;
      const uint32_t ntiles = pd.nI_pad / kTileN;
      const uint32_t qb = n_qbuf == 2 ? (qi & 1u) : 0u;
      const uint32_t quse = n_qbuf == 2 ? (qi >> 1) : qi;
      mbar_wait(bar_qempty + 8 * qb, (quse & 1u) ^ 1u);
      if (elect_one()) {
        mbar_arrive_expect_tx(bar_qfull + 8 * qb, nkb * kBoxBytes);
        for (uint32_t kb = 0; kb < nkb; ++kb)
          tma_load_2d(q_base + qb * q_bytes + kb * kBoxBytes, mq, (int)(kb * kKBlock), (int)(wi.sb * kTileRows),
                      bar_qfull + 8 * qb);
      }
      __syncwarp();
      for (uint32_t t = 0; t < ntiles; ++t) {
        for (uint32_t kb = 0; kb < nkb; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1u);
          if (elect_one()) {
            const uint32_t dst = d_base + stage * kStageBytes;
            mbar_arrive_expect_tx(bar_full + 8 * stage, kStageBytes);
            tma_load_2d(dst, md, (int)(kb * kKBlock), (int)(t * kTileN), bar_full + 8 * stage);
            tma_load_2d(dst + kBoxBytes, md, (int)(kb * kKBlock), (int)(t * kTileN + kTileRows), bar_full + 8 * stage);
          }
          __syncwarp();
          if (++stage == n_stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // =========================================== consumers ===========================================
  setmaxnreg_inc<232>();
  const uint32_t cw = wg - 1u;                                   // query rows [64 cw, 64 cw + 64) of the block
  const uint32_t q = lane & 3u;                                  // lane inside the quad
  const uint32_t row0 = cw * 64u + (warp & 3u) * 16u + (lane >> 2);  // accumulator rows row0 and row0 + 8
  uint32_t stage = 0, phase = 0, qi = 0;
  float acc[128];
  for (uint32_t it = blockIdx.x; it < n_items; it += gridDim.x, ++qi) {
    const WorkItem wi = items[it];
    const PairDesc pd = pairs[wi.pair];
    const uint32_t ntiles = pd.nI_pad / kTileN;
    const uint32_t qb = n_qbuf == 2 ? (qi & 1u) : 0u;
    const uint32_t qf = (n_qbuf == 2 ? (qi >> 1) : qi) & 1u;
    const uint32_t keep_mask = ~((1u << pd.chunk_bits) - 1u);
    float key0[kNumKeys], key1[kNumKeys];
#pragma unroll
    for (int i = 0; i < kNumKeys; ++i) key0[i] = key1[i] = __uint_as_float(kKeySentinel);
    const uint32_t a_base = q_base + qb * q_bytes + cw * (kBoxBytes / 2);  // 64 rows x 128 B into each query box
    mbar_wait(bar_qfull + 8 * qb, qf);
    for (uint32_t t = 0; t < ntiles; ++t) {
      uint32_t ks_left = ksteps, prev = 0;
      for (uint32_t kb = 0; kb < nkb; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        wgmma_fence();
        const uint32_t a_lo = desc_lo(a_base + kb * kBoxBytes);
        const uint32_t b_lo = desc_lo(d_base + stage * kStageBytes);
        const uint32_t ks_here = ks_left < 4u ? ks_left : 4u;
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
          if (k < ks_here) wgmma_m64n256k16(acc, make_desc(a_lo + 2 * k), make_desc(b_lo + 2 * k), (kb | k) != 0u ? 1u : 0u);
        }
        wgmma_commit();
        if (kb > 0) {  // the previous K-block's MMAs have read their stage
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
        }
        prev = stage;
        ks_left -= ks_here;
        if (++stage == n_stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      if (lane == 0) {
        mbar_arrive(bar_empty + 8 * prev);
        if (t + 1 == ntiles) mbar_arrive(bar_qempty + 8 * qb);  // every MMA of the item has read the query block
      }
      // accumulator column 8 j + 2 q + {0, 1} of rows row0 / row0 + 8 is acc[4 j + {0, 1}] / acc[4 j + {2, 3}];
      // column c of the tile is database row t * 256 + c, i.e. chunk t * 32 + c / 8
      const uint32_t chunk0 = t * (kTileN / kChunk);
#pragma unroll
      for (uint32_t g = 0; g < 8; ++g) {
        const float* a = acc + 16 * g;
        const float m0 = quad_min4(fminf(a[0], a[1]), fminf(a[4], a[5]), fminf(a[8], a[9]), fminf(a[12], a[13]), q);
        const float m1 = quad_min4(fminf(a[2], a[3]), fminf(a[6], a[7]), fminf(a[10], a[11]), fminf(a[14], a[15]), q);
        key_insert<true>(m0, chunk0 + 4 * g + q, keep_mask, key0);
        key_insert<true>(m1, chunk0 + 4 * g + q, keep_mask, key1);
      }
    }
    // the four lanes of a quad hold the keys of disjoint chunk sets of the same two rows
    merge_keys(key0, 1);
    merge_keys(key0, 2);
    merge_keys(key1, 1);
    merge_keys(key1, 2);
    if (q < 2) {
      float k[kNumKeys];
#pragma unroll
      for (int i = 0; i < kNumKeys; ++i) k[i] = q == 0 ? key0[i] : key1[i];
      const uint32_t row = wi.sb * kTileRows + row0 + 8u * q;
      uint4 o0, o1;
      o0.x = __float_as_uint(k[0]); o0.y = __float_as_uint(k[1]);
      o0.z = __float_as_uint(k[2]); o0.w = __float_as_uint(k[3]);
      o1.x = __float_as_uint(k[4]); o1.y = __float_as_uint(k[5]);
      o1.z = kKeySentinel; o1.w = kKeySentinel;
      uint4* dst = (uint4*)keys_out + (size_t)(pd.q_ofs + row) * (kKeyStride / 4);
      dst[0] = o0;
      dst[1] = o1;
    }
  }
}

static int ring_stages(int nkb, int n_qbuf) {
  const size_t fixed = 1024 + 8 * (2 * kMaxStages + 4) + (size_t)n_qbuf * nkb * kBoxBytes;
  const int stages = (int)((kSmemOptIn - fixed) / kStageBytes);
  return stages > kMaxStages ? kMaxStages : stages;
}

int launch_l2_candidates(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const WorkItem* d_items,
                         uint32_t n_items, uint32_t* d_keys, int kp_cols, int ksteps) {
  if (n_items == 0) return R3D_OK;
  const int nkb = (kp_cols + kKBlock - 1) / kKBlock;
  if (nkb > kMaxKBlocks) return fail(ctx, R3D_ERR_UNSUPPORTED, "descriptor dimension too large for the tensor-core path");
  const int n_qbuf = ring_stages(nkb, 2) >= 3 ? 2 : 1;  // very wide descriptors: keep the ring deep enough instead
  const int stages = ring_stages(nkb, n_qbuf);
  const size_t smem = 1024 + (size_t)n_qbuf * nkb * kBoxBytes + (size_t)stages * kStageBytes + 8 * (2 * kMaxStages + 4);
  R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(k_l2_candidates, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const uint32_t grid = n_items < (uint32_t)w.sm_count ? n_items : (uint32_t)w.sm_count;
  k_l2_candidates<<<grid, kThreads, smem, w.stream>>>((const CUtensorMap*)w.d_tmapQ, (const CUtensorMap*)w.d_tmapD,
                                                      d_pairs, d_items, n_items, d_keys, (uint32_t)nkb, (uint32_t)ksteps,
                                                      (uint32_t)stages, (uint32_t)n_qbuf);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

}  // namespace r3d
