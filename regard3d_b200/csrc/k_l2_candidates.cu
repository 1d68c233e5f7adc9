// k_l2_candidates.cu -- the tensor-core candidate kernel (sm_90a: TMA, mbarrier, wgmma).
//
// Work item = (pair, query block of view J: 128 rows on the fp16 path, 256 on the integer path).  For every query row
// the kernel evaluates a squared distance against all database rows of view I and keeps the kNumKeys smallest chunk
// minima (kChunk consecutive database rows each), packed with the chunk id, in keys_out.  Two operand kinds, one
// kernel template:
//   fp16 (kU8 = false)  the distance surrogate opQ(J) . opD(I) of the fp16 operands (k_view_prepare), f32 accumulation
//   u8   (kU8 = true)   uint8 descriptors read in place (int_operand()): ||a||^2 - 2 q.a from u8 x u8 -> s32 MMAs plus
//                       the exact norms, so the keys are exact up to the chunk-id packing
//
// Persistent CTAs (one per SM, 227 KB of shared memory), one producer and kConsumers consumer warpgroups:
//   warpgroup 0      one TMA producer warp: the item's query block (kConsumers / 2 boxes of 128 rows x 128 bytes per
//                    K-block, double buffered across items) and a ring of database stages (one 128-byte K-block of a
//                    256-row tile; u8: plus the tile's 256 database norms)
//   warpgroup 1 + c  consumer of query rows [64 c, 64 c + 64) of the block: the MMAs, then the chunk minima and the key
//                    insertion in registers.
//     fp16: 2 consumers (the 128-register f32 accumulator leaves no room for more); per 256-row tile, m64n256k16,
//           then the epilogue.
//     u8:   4 consumers, so every database tile in shared memory feeds 256 query rows; per 128-row half tile,
//           m64n128k32 (the K extent fixed at compile time: back-to-back MMAs, no branch) into one 64-register s32
//           accumulator.  The chunk minima of a half are taken from the accumulator as soon as its MMAs are done; the
//           next half's MMAs are issued, and the half's key insertion runs behind them.  The other three consumers
//           keep MMAs in the tensor pipe too.  The database map loads every 32-row group with its row pairs
//           transposed (context.cu), so each lane of a quad holds whole chunks: the chunk minima take no shuffle.  An
//           integer bound taken once per tile from the quad's four sets of a row rejects nearly every chunk before its
//           key is formed; the rest are inserted in warp-uniform rounds, one round loop per set.
// Barriers: full[s] (TMA bytes landed), empty[s] (every consumer warp is done with the stage), qfull / qempty the same
// for the query buffers.
#include "r3d_internal.cuh"
#include "tc_ptx.cuh"

namespace r3d {

using namespace tcx;

namespace {

constexpr int kMaxStages = 8;
constexpr uint32_t kTileN = 256;                  // database rows per tile (the wgmma N extent)
constexpr uint32_t kStageBytes = 2 * kBoxBytes;   // one K-block of a 256-row tile: two 128-row TMA boxes
constexpr uint32_t kNormBytes = kTileN * 4;       // u8: the int32 norms of a tile's database rows
constexpr uint32_t kConsumersF16 = kTileRows / 64;  // consumer warpgroups (64 query rows each) of the fp16 path
constexpr uint32_t kConsumersU8 = kSuperRows / 64;  // ... and of the integer path
constexpr size_t kSmemOptIn = 232448;             // 227 KB: the largest dynamic shared memory of one block on sm_90
static_assert(kChunk == 8, "the epilogue reduces one 8-column block of the wgmma accumulator per chunk");

// fp16: minima of four consecutive chunks of one accumulator row, spread over the 4 lanes of a quad (2 columns each),
// reduced and scattered so that lane q of the quad ends with the minimum of chunk q: 3 shuffles for 4 chunks.
__device__ __forceinline__ float quad_min4(float p0, float p1, float p2, float p3, uint32_t q) {
  const bool b1 = (q & 2u) != 0, b0 = (q & 1u) != 0;
  const float k0 = fminf(b1 ? p2 : p0, __shfl_xor_sync(0xffffffffu, b1 ? p0 : p2, 2));
  const float k1 = fminf(b1 ? p3 : p1, __shfl_xor_sync(0xffffffffu, b1 ? p1 : p3, 2));
  return fminf(b0 ? k1 : k0, __shfl_xor_sync(0xffffffffu, b0 ? k0 : k1, 1));
}

// u8: the minimum of one chunk, held whole by one lane (3 VIMNMX3 + 1 VIMNMX)
__device__ __forceinline__ int32_t min8(const int32_t (&v)[8]) {
  return __vimin3_s32(__vimin3_s32(v[0], v[1], v[2]), __vimin3_s32(v[3], v[4], v[5]), min(v[6], v[7]));
}

// u8: the packed key of a chunk whose bracket minimum (min of ||a||^2 - 2 q.a) is m; exact: real distances are < 2^24
__device__ __forceinline__ float chunk_key(int32_t m, int32_t qn, uint32_t cid, uint32_t keep_mask) {
  return __uint_as_float((__float_as_uint((float)(m + qn)) & keep_mask) | cid);
}

// u8: an integer bound on the bracket minima whose keys can be below kmax.  Such a key's bits above the chunk bits are
// at most those of kmax, so its distance converts to a float below F = ((kmax & keep_mask) + 2^chunk_bits) as bits.
// Rounding to nearest is monotone and F is a float, so every integer distance >= F converts to a float >= F:
// m + qn <= ceil(F) - 1 keeps every chunk that can enter the set (and a few that cannot: the network drops those).
// F is +inf while the set holds the FLT_MAX sentinel; the conversion saturates to INT_MAX there.
// Returned as ~bound = qn - ceil(F), so that m passes exactly when m + ~bound is negative.
__device__ __forceinline__ int32_t bracket_bound_not(float kmax, uint32_t keep_mask, int32_t qn) {
  const float f = __uint_as_float((__float_as_uint(kmax) & keep_mask) - keep_mask);  // - keep_mask = + 2^chunk_bits
  return qn - __float2int_ru(f);
}

// u8: an upper bound on the kNumKeys-th smallest key of the union of the quad's four sets of one row: the smallest of
// their largest keys, or the largest of their second keys (eight keys are at or below it).  The FLT_MAX sentinels are
// equal, but a bound below FLT_MAX is the largest key of a full set or the largest of eight real keys, which differ.
__device__ __forceinline__ float quad_bound(const float (&key)[kNumKeys]) {
  float k5 = key[kNumKeys - 1], k1 = key[1];
#pragma unroll
  for (int d = 1; d <= 2; d *= 2) {
    k5 = fminf(k5, __shfl_xor_sync(0xffffffffu, k5, d));
    k1 = fmaxf(k1, __shfl_xor_sync(0xffffffffu, k1, d));
  }
  return fminf(k5, k1);
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

// kKSteps: u8, the k32 steps of the descriptor (ceil(D / 32), so ceil(kKSteps / 4) K-blocks); 0 on the fp16 path,
// which takes nkb and ksteps at run time.
template <bool kU8, uint32_t kConsumers, uint32_t kKSteps>
__global__ void __launch_bounds__(128 * (kConsumers + 1), 1)
k_l2_candidates(const CUtensorMap* __restrict__ tmapQ, const CUtensorMap* __restrict__ tmapD,
                const PairDesc* __restrict__ pairs, const WorkItem* __restrict__ items, uint32_t n_items,
                uint32_t* __restrict__ keys_out, uint32_t nkb, uint32_t ksteps, uint32_t n_stages, uint32_t n_qbuf) {
  static_assert(kConsumers == 2 || (kU8 && kConsumers == 4), "fp16: 2 consumers; u8: 2 or 4");
  static_assert(kU8 ? (kKSteps >= 1 && kKSteps <= 8) : kKSteps == 0, "u8: 1 .. 8 k32 steps (D <= 256); fp16: 0");
  constexpr uint32_t kBoxCols = kU8 ? 128u : (uint32_t)kKBlock;  // elements in a 128-byte box row
  constexpr uint32_t kQBoxes = kConsumers / 2;                   // 128-row query boxes per K-block
  constexpr uint32_t kBlockRows = kQBoxes * kTileRows;           // query rows per work item
  constexpr uint32_t kConsumerWarps = 4 * kConsumers;
  // Register split (setmaxnreg): 640 threads launch with at most 96 registers each (65536 / 640, in steps of 8), and
  // the consumers can only take what the producer warpgroup gives back: 128 x 24 + 512 x 112 <= 640 x 96.  384
  // threads launch with 168: 128 x 40 + 256 x 232 = 384 x 168.
  constexpr uint32_t kProducerRegs = kConsumers == 4 ? 24u : 40u;
  constexpr uint32_t kConsumerRegs = kConsumers == 4 ? 112u : 232u;
  extern __shared__ unsigned char smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  // n_qbuf (1 or 2) x kQBoxes x nkb boxes ([buffer][box][K-block]): the item's query rows.  With two buffers the next
  // item's query block is loaded while the current item's last tiles are still in the tensor pipe.
  const uint32_t q_base = base;
  const uint32_t q_bytes = kQBoxes * nkb * kBoxBytes;
  const uint32_t d_base = q_base + n_qbuf * q_bytes;            // n_stages stages
  const uint32_t n_base = d_base + n_stages * kStageBytes;      // u8: n_stages x kNormBytes
  const uint32_t bar_full = n_base + (kU8 ? n_stages * kNormBytes : 0u);  // [kMaxStages]
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
    setmaxnreg_dec<kProducerRegs>();
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
        mbar_arrive_expect_tx(bar_qfull + 8 * qb, q_bytes);
#pragma unroll
        for (uint32_t b = 0; b < kQBoxes; ++b)  // rows past the view are zero-filled
          for (uint32_t kb = 0; kb < nkb; ++kb)
            tma_load_2d(q_base + qb * q_bytes + (b * nkb + kb) * kBoxBytes, mq, (int)(kb * kBoxCols),
                        (int)(wi.sb * kBlockRows + b * kTileRows), bar_qfull + 8 * qb);
      }
      __syncwarp();
      for (uint32_t t = 0; t < ntiles; ++t) {
        for (uint32_t kb = 0; kb < nkb; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1u);
          if (elect_one()) {
            const uint32_t dst = d_base + stage * kStageBytes;
            const bool norms = kU8 && kb == 0;  // the tile's norms travel with its first K-block
            mbar_arrive_expect_tx(bar_full + 8 * stage, kStageBytes + (norms ? kNormBytes : 0u));
            if constexpr (kU8) {  // the permuted database map (context.cu): 4 groups of 32 rows per box
              constexpr uint32_t kGroupsPerBox = kTileRows / kGroupRows;
              tma_load_5d(dst, md, (int)(kb * kBoxCols), 0, 0, 0, (int)(t * 2 * kGroupsPerBox), bar_full + 8 * stage);
              tma_load_5d(dst + kBoxBytes, md, (int)(kb * kBoxCols), 0, 0, 0, (int)(t * 2 * kGroupsPerBox + kGroupsPerBox),
                          bar_full + 8 * stage);
            } else {
              tma_load_2d(dst, md, (int)(kb * kBoxCols), (int)(t * kTileN), bar_full + 8 * stage);
              tma_load_2d(dst + kBoxBytes, md, (int)(kb * kBoxCols), (int)(t * kTileN + kTileRows), bar_full + 8 * stage);
            }
            if (norms) bulk_load(n_base + stage * kNormBytes, pd.normI + t * kTileN, kNormBytes, bar_full + 8 * stage);
          }
          __syncwarp();
          if (++stage == n_stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // =========================================== consumers ===========================================
  setmaxnreg_inc<kConsumerRegs>();
  const uint32_t cw = wg - 1u;                                   // query rows [64 cw, 64 cw + 64) of the block
  const uint32_t q = lane & 3u;                                  // lane inside the quad
  const uint32_t row0 = cw * 64u + (warp & 3u) * 16u + (lane >> 2);  // accumulator rows row0 and row0 + 8
  uint32_t stage = 0, phase = 0, qi = 0;
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
    // box cw / 2 of each K-block, 64 rows x 128 B into it
    const uint32_t a_base = q_base + qb * q_bytes +
                            (kQBoxes == 1 ? cw * (kBoxBytes / 2) : (cw >> 1) * nkb * kBoxBytes + (cw & 1u) * (kBoxBytes / 2));
    if constexpr (kU8) {
      // ||q||^2 of the two rows (kPadNorm beyond nJ: those rows' keys are never read)
      const int32_t qn0 = __ldg(pd.normJ + wi.sb * kBlockRows + row0);
      const int32_t qn1 = __ldg(pd.normJ + wi.sb * kBlockRows + row0 + 8u);
      int32_t acc[64];
      constexpr uint32_t kNkb = (kKSteps + 3) / 4;
      // The low descriptor words of the consumer's query rows (K-block 0) and of the ring (stage 0, half 0), taken
      // once per item from a warp-uniform consumer index, so they and everything derived from them stay in uniform
      // registers.  Shared-memory addresses are below 2^18 bytes, so the 14-bit start-address field of a descriptor
      // never carries: K-block kb, stage s, half h and k-step k only add (kb * kBoxBytes + s * kStageBytes +
      // h * kBoxBytes) / 16 + 2 k.
      const uint32_t cw_u = __shfl_sync(0xffffffffu, cw, 0);
      const uint32_t a_lo = desc_lo(q_base + qb * q_bytes +
                                    (kQBoxes == 1 ? cw_u * (kBoxBytes / 2)
                                                  : (cw_u >> 1) * nkb * kBoxBytes + (cw_u & 1u) * (kBoxBytes / 2)));
      const uint32_t d_lo = desc_lo(d_base);
      // MMAs of half h (database rows h * 128 .. + 127) of the tile whose K-blocks start at stage s0: kKSteps
      // back-to-back m64n128k32 behind one fence, no branch
      auto issue = [&](uint32_t h, uint32_t s0) {
        wgmma_fence();
        uint32_t s = s0;
#pragma unroll
        for (uint32_t kb = 0; kb < kNkb; ++kb) {
          const uint32_t b_lo = d_lo + (s * kStageBytes + h * kBoxBytes) / 16u;
#pragma unroll
          for (uint32_t k = 0; k < 4 && 4 * kb + k < kKSteps; ++k)
            wgmma_m64n128k32_u8(acc, make_desc(a_lo + kb * (kBoxBytes / 16u) + 2 * k), make_desc(b_lo + 2 * k),
                                (kb | k) != 0u ? 1u : 0u);
          if (kb + 1 < kNkb && ++s == n_stages) s = 0;
        }
        wgmma_commit();
      };
      // Accumulator column 8 j + 2 q + {0, 1} of rows row0 / row0 + 8 is acc[4 j + {0, 1}] / acc[4 j + {2, 3}].  The
      // database map permutes every 32-row group (context.cu): column 32 g + 8 jj + 2 q + e of half h of tile t holds
      // database row t * 256 + h * 128 + 32 g + 8 q + 2 jj + e.  So the 8 columns of lane q in group g (j = 4 g + jj)
      // are the 8 rows of chunk t * 32 + h * 16 + 4 g + q, and their norms are 8 consecutive words of shared memory.
      // ||q - a||^2 = ||q||^2 + (||a||^2 - 2 q.a): each lane takes the minima of its chunks over the bracket, exactly
      // in s32 and without leaving its registers.
      // The item writes the kNumKeys smallest keys of the union of the quad's four sets (merge_keys), so a chunk whose
      // key is not below U, any upper bound on the union's kNumKeys-th smallest key, can be dropped: it is not in the
      // row's final keys, and every chunk that is passes U and stays among its own set's kNumKeys smallest.  Keys
      // only fall, so a U taken earlier stays valid.  Once per tile, in the first half, after the previous half's
      // insertion, quad_bound takes U from the four sets and bracket_bound_not turns it into an integer bound on the
      // bracket minimum; the second half reuses it.  A chunk costs one add (the sign of m + ~bound says whether it
      // passes) and its key is only formed in an insertion round.  Inserting a chunk whose key is above U, passed or
      // failed, is harmless: it can only push out keys above its own, which are not among the row's final keys.  So
      // the rounds below may insert chunks that failed, and the merged keys do not depend on the order of insertion
      // (the keys of a row differ in their chunk bits).
      // take_minima reads the accumulator and the half's norms; insert reads neither, so it runs while the MMAs of the
      // next half write the accumulator.
      int32_t m0[4], m1[4];
      int32_t nb0, nb1;  // ~bound of each set for the current tile
      // The insertion order of each set's four chunks, highest bit first: bit 16 + 4 g + 3 for a chunk g that passed
      // the bound, bit 4 g + 3 for one that failed.  Bits 2 and 3 of a bit's index are g.
      uint32_t u0, u1;
      auto take_minima = [&](uint32_t h, uint32_t s0) {
        const int32_t* nrm = (const int32_t*)(smem_raw + (n_base + s0 * kNormBytes - smem_u32(smem_raw))) + h * 128u + 8u * q;
        if (h == 0) {
          nb0 = bracket_bound_not(quad_bound(key0), keep_mask, qn0);
          nb1 = bracket_bound_not(quad_bound(key1), keep_mask, qn1);
        }
#pragma unroll
        for (uint32_t g = 0; g < 4; ++g) {
          const int4 na = *(const int4*)(nrm + kGroupRows * g);
          const int4 nb = *(const int4*)(nrm + kGroupRows * g + 4);
          const int32_t* a = acc + 16 * g;
          const int32_t d0[8] = {na.x - 2 * a[0], na.y - 2 * a[1], na.z - 2 * a[4], na.w - 2 * a[5],
                                 nb.x - 2 * a[8], nb.y - 2 * a[9], nb.z - 2 * a[12], nb.w - 2 * a[13]};
          const int32_t d1[8] = {na.x - 2 * a[2], na.y - 2 * a[3], na.z - 2 * a[6], na.w - 2 * a[7],
                                 nb.x - 2 * a[10], nb.y - 2 * a[11], nb.z - 2 * a[14], nb.w - 2 * a[15]};
          m0[g] = min8(d0);
          m1[g] = min8(d1);
        }
        // the top nibble of m[g] + ~bound to nibble g (its sign to bit 4 g + 3), one funnel shift per chunk; no
        // overflow: m + ~bound = (m + qn) - ceil(F) with 0 <= m + qn <= 2^28 + 2^23 and 16 <= ceil(F) <= INT_MAX
        uint32_t w0 = 0, w1 = 0;
#pragma unroll
        for (int g = 3; g >= 0; --g) {
          w0 = __funnelshift_l((uint32_t)(m0[g] + nb0), w0, 4);
          w1 = __funnelshift_l((uint32_t)(m1[g] + nb1), w1, 4);
        }
        w0 &= 0x8888u;
        w1 &= 0x8888u;
        u0 = w0 << 16 | (w0 ^ 0x8888u);
        u1 = w1 << 16 | (w1 ^ 0x8888u);
      };
      // One warp-uniform round loop per set: per round every lane inserts the set's next chunk, until no lane of the
      // warp has a chunk that passed left, so a set in which no lane's chunk passed costs one vote.  A lane with fewer
      // such chunks inserts chunks that failed, which is harmless (above).  No chunk is inserted twice, and a set has
      // four chunks and at most four rounds run, so no sentinel is needed.
      auto next_key = [&](uint32_t& u, const int32_t (&m)[4], int32_t qn, uint32_t chunk0) {
        const uint32_t i = 31 - __clz(u);
        uint32_t below;  // (1 << i) - 1 in one BMSK: clears u's highest bit
        asm("bmsk.clamp.b32 %0, 0, %1;" : "=r"(below) : "r"(i));
        u &= below;
        const int32_t lo = (i & 4u) ? m[1] : m[0];
        const int32_t hi = (i & 4u) ? m[3] : m[2];
        return chunk_key((i & 8u) ? hi : lo, qn, chunk0 | (i & 12u), keep_mask);
      };
      auto insert = [&](uint32_t t, uint32_t h) {
        const uint32_t chunk0 = t * (kTileN / kChunk) + h * (kTileN / 2 / kChunk) + q;  // bits 2 and 3 clear
        while (__any_sync(0xffffffffu, u0 >> 16 != 0u)) key_insert_packed(next_key(u0, m0, qn0, chunk0), key0);
        while (__any_sync(0xffffffffu, u1 >> 16 != 0u)) key_insert_packed(next_key(u1, m1, qn1, chunk0), key1);
      };
      // the first stage of the next tile, once all of its K-blocks have landed
      auto wait_tile = [&]() {
        const uint32_t s0 = stage;
#pragma unroll
        for (uint32_t kb = 0; kb < kNkb; ++kb) {
          mbar_wait(bar_full + 8 * stage, phase);
          if (++stage == n_stages) { stage = 0; phase ^= 1u; }
        }
        return s0;
      };
      auto mma_done = [&]() {
        wgmma_wait<0>();
        wgmma_fence_operand(acc);
      };
      // One accumulator, and the insertions of each half behind the MMAs of the next: per half, wait for its MMAs, take
      // its minima, issue the next half's MMAs, then insert.  The halves are unrolled, so each has its own wait.  The
      // item's last half is inserted with nothing in flight.  take_minima of a half runs after the previous half's
      // insert, so every bound is taken from the same keys as with no overlap.  Views are padded to whole tiles
      // (n_pad >= 256), so an item has at least one tile.
      mbar_wait(bar_qfull + 8 * qb, qf);
      uint32_t s_t = wait_tile();
      issue(0, s_t);
      mma_done();
      take_minima(0, s_t);
      for (uint32_t t = 0;; ++t) {
        issue(1, s_t);
        insert(t, 0);
        mma_done();
        take_minima(1, s_t);
        // the tile's norms and operands are read: hand its stages back to the producer
        __syncwarp();
        if (lane == 0)
#pragma unroll
          for (uint32_t kb = 0, s = s_t; kb < kNkb; ++kb) {
            mbar_arrive(bar_empty + 8 * s);
            if (++s == n_stages) s = 0;
          }
        if (t + 1 == ntiles) {
          // every MMA of the item has read the query block
          if (lane == 0) mbar_arrive(bar_qempty + 8 * qb);
          insert(t, 1);
          break;
        }
        s_t = wait_tile();
        issue(0, s_t);
        insert(t, 1);
        mma_done();
        take_minima(0, s_t);
      }
    } else {
      float acc[128];
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
      const uint32_t row = wi.sb * kBlockRows + row0 + 8u * q;
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

static int ring_stages(uint32_t q_bytes, int n_qbuf, uint32_t stage_bytes) {
  const size_t fixed = 1024 + 8 * (2 * kMaxStages + 4) + (size_t)n_qbuf * q_bytes;
  const int stages = (int)((kSmemOptIn - fixed) / stage_bytes);
  return stages > kMaxStages ? kMaxStages : stages;
}

int launch_l2_candidates(r3d_ctx* ctx, DeviceWorker& w, const PairDesc* d_pairs, const WorkItem* d_items,
                         uint32_t n_items, uint32_t* d_keys, int dtype, uint32_t dim) {
  if (n_items == 0) return R3D_OK;
  const bool u8 = int_operand(dtype, dim);
  // u8: 128 columns per K-block, k32 steps; fp16: Kp = operand_cols(dim) columns, 64 per K-block, k16 steps
  const int nkb = u8 ? ((int)dim + 127) / 128 : (operand_cols((int)dim) + kKBlock - 1) / kKBlock;
  const int ksteps = u8 ? ((int)dim + 31) / 32 : operand_ksteps((int)dim);
  if (nkb > kMaxKBlocks) return fail(ctx, R3D_ERR_UNSUPPORTED, "descriptor dimension too large for the tensor-core path");
  const uint32_t consumers = u8 ? kConsumersU8 : kConsumersF16;
  const uint32_t stage_bytes = kStageBytes + (u8 ? kNormBytes : 0u);
  const uint32_t q_bytes = consumers / 2 * nkb * kBoxBytes;  // one query buffer: the item's query rows, nkb K-blocks
  // The four u8 consumers can be a tile apart: the ring needs two tiles.  Two query buffers when the ring keeps that
  // depth, else one (very wide descriptors).  u8, 33 KB stages: D <= 128 (nkb = 1) 2 x 32 KB of queries and 4 stages;
  // D = 256 (nkb = 2) 2 x 64 KB would leave 2 stages, so 1 x 64 KB and 4 stages (two tiles).
  const int min_stages = u8 ? 2 * nkb : 3;
  const int n_qbuf = ring_stages(q_bytes, 2, stage_bytes) >= min_stages ? 2 : 1;
  const int stages = ring_stages(q_bytes, n_qbuf, stage_bytes);
  const size_t smem = 1024 + (size_t)n_qbuf * q_bytes + (size_t)stages * stage_bytes + 8 * (2 * kMaxStages + 4);
  using Kernel = decltype(&k_l2_candidates<false, kConsumersF16, 0>);
  // u8: the K extent is a template parameter, so each consumer issues its k32 steps back to back without a branch
  static const Kernel kU8Kernels[8] = {
      k_l2_candidates<true, kConsumersU8, 1>, k_l2_candidates<true, kConsumersU8, 2>, k_l2_candidates<true, kConsumersU8, 3>,
      k_l2_candidates<true, kConsumersU8, 4>, k_l2_candidates<true, kConsumersU8, 5>, k_l2_candidates<true, kConsumersU8, 6>,
      k_l2_candidates<true, kConsumersU8, 7>, k_l2_candidates<true, kConsumersU8, 8>};
  const Kernel kern = u8 ? kU8Kernels[ksteps - 1] : k_l2_candidates<false, kConsumersF16, 0>;
  R3D_CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const uint32_t grid = n_items < (uint32_t)w.sm_count ? n_items : (uint32_t)w.sm_count;
  kern<<<grid, 128 * (consumers + 1), smem, w.stream>>>((const CUtensorMap*)w.d_tmapQ, (const CUtensorMap*)w.d_tmapD, d_pairs, d_items,
                                           n_items, d_keys, (uint32_t)nkb, (uint32_t)ksteps, (uint32_t)stages,
                                           (uint32_t)n_qbuf);
  R3D_CUDA_TRY(ctx, cudaGetLastError());
  return R3D_OK;
}

}  // namespace r3d
