// threefry2x32 (20 rounds), the counter-based generator of jax.random (viettts_b200/jaxrng.py restates it on the host):
// the acoustic model's reference dropout masks (nat.cu) and the watermark's chips (watermark.cu).
#pragma once

#include <cstdint>

__host__ __device__ inline void threefry2x32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t& o0, uint32_t& o1) {
  const uint32_t ks2 = 0x1BD11BDAu ^ k0 ^ k1;
  uint32_t x0 = c0 + k0, x1 = c1 + k1;
  const int R0[4] = {13, 15, 26, 6}, R1[4] = {17, 29, 16, 24};
  const uint32_t ks[3] = {k0, k1, ks2};
#pragma unroll
  for (int blk = 0; blk < 5; ++blk) {
    const int* R = (blk & 1) ? R1 : R0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      x0 += x1;
      x1 = (x1 << R[r]) | (x1 >> (32 - R[r]));
      x1 ^= x0;
    }
    x0 += ks[(blk + 1) % 3];
    x1 += ks[(blk + 2) % 3] + (uint32_t)(blk + 1);
  }
  o0 = x0;
  o1 = x1;
}
