// acransac_rng.cuh -- the sample stream of ACRANSAC on the device.
//
// robust_estimation/rand_sampling.hpp UniformSample() draws with `std::mt19937` (default seed, one generator per
// ACRANSAC call) and `std::uniform_int_distribution<uint32_t>(i, last)`.  mt19937 is fully specified by the C++
// standard ([rand.predef]: the 10000th value of a default-constructed engine is 4123659995).  The distribution is
// implementation-defined; what is restated here is libstdc++'s (GCC >= 11, bits/uniform_int_dist.h): for a 32-bit
// generator and a range below 2^32 it is Lemire's nearly-divisionless method on a 64-bit product
//     product = g() * range;  low = (uint32) product;
//     if (low < range) { threshold = -range % range; while (low < threshold) { product = g() * range; low = ...; } }
//     return (product >> 32) + a;
// and for the full range simply g().  rng_selftest() (acransac_fused.cu) checks this restatement against the host's own
// <random> once per process; when the two disagree (another standard library) every AC-RANSAC entry point returns
// R3D_ERR_UNSUPPORTED (AcFused::plan), so results never depend on this file being right for an unknown library.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define R3D_RNG_HD __host__ __device__ __forceinline__
#else
#define R3D_RNG_HD inline
#endif

namespace r3d {

constexpr int kMtN = 624, kMtM = 397;

struct Mt19937 {  // state lives wherever the caller puts it (shared memory on the device)
  uint32_t x[kMtN];
  uint32_t idx;
};

R3D_RNG_HD void mt_seed(Mt19937& s, uint32_t seed = 5489u) {
  s.x[0] = seed;
  for (int i = 1; i < kMtN; ++i) s.x[i] = 1812433253u * (s.x[i - 1] ^ (s.x[i - 1] >> 30)) + (uint32_t)i;
  s.idx = kMtN;
}

R3D_RNG_HD void mt_twist(Mt19937& s) {
  for (int k = 0; k < kMtN; ++k) {
    const uint32_t y = (s.x[k] & 0x80000000u) | (s.x[(k + 1) % kMtN] & 0x7fffffffu);
    s.x[k] = s.x[(k + kMtM) % kMtN] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
  }
  s.idx = 0;
}

R3D_RNG_HD uint32_t mt_next(Mt19937& s) {
  if (s.idx >= (uint32_t)kMtN) mt_twist(s);
  uint32_t y = s.x[s.idx++];
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}

// std::uniform_int_distribution<uint32_t>(a, b)(g), libstdc++; counts the generator outputs it consumed
R3D_RNG_HD uint32_t uniform_u32(Mt19937& s, uint32_t a, uint32_t b, uint32_t* used) {
  const uint32_t urange = b - a;
  if (urange == 0xffffffffu) {
    ++*used;
    return mt_next(s);
  }
  const uint32_t range = urange + 1u;
  uint64_t product = (uint64_t)mt_next(s) * (uint64_t)range;
  ++*used;
  uint32_t low = (uint32_t)product;
  if (low < range) {
    const uint32_t threshold = (0u - range) % range;
    while (low < threshold) {
      product = (uint64_t)mt_next(s) * (uint64_t)range;
      ++*used;
      low = (uint32_t)product;
    }
  }
  return (uint32_t)(product >> 32) + a;
}

// host-side check of the restatement against the process's <random> (defined in acransac_fused.cu)
bool rng_selftest();

}  // namespace r3d
