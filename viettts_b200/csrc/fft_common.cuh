// Register-resident building blocks of the warp FFT-1024 (four-step 1024 = 32 x 32) shared by MelFilter (melspec.cu)
// and the bias denoiser (denoise.cu): complex product, the 32-point twiddles as immediates, and the in-register
// 32-point DFT.
#pragma once

#include <cuda_runtime.h>

namespace fftc {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// exp(-2 pi i k / 32), k = 0..15; k is a compile-time constant at every call site (fully unrolled loops)
__device__ __forceinline__ float2 w32(int k) {
  switch (k) {
    case 0: return make_float2(1.f, 0.f);
    case 1: return make_float2(0.98078528040323043f, -0.19509032201612825f);
    case 2: return make_float2(0.92387953251128674f, -0.38268343236508978f);
    case 3: return make_float2(0.83146961230254524f, -0.55557023301960218f);
    case 4: return make_float2(0.70710678118654757f, -0.70710678118654757f);
    case 5: return make_float2(0.55557023301960229f, -0.83146961230254524f);
    case 6: return make_float2(0.38268343236508984f, -0.92387953251128674f);
    case 7: return make_float2(0.19509032201612833f, -0.98078528040323043f);
    case 8: return make_float2(0.f, -1.f);
    case 9: return make_float2(-0.19509032201612819f, -0.98078528040323043f);
    case 10: return make_float2(-0.38268343236508973f, -0.92387953251128674f);
    case 11: return make_float2(-0.55557023301960196f, -0.83146961230254546f);
    case 12: return make_float2(-0.70710678118654746f, -0.70710678118654757f);
    case 13: return make_float2(-0.83146961230254535f, -0.55557023301960218f);
    case 14: return make_float2(-0.92387953251128674f, -0.38268343236508989f);
    default: return make_float2(-0.98078528040323043f, -0.19509032201612861f);
  }
}

__host__ __device__ constexpr int bitrev5(int x) {
  return ((x & 1) << 4) | ((x & 2) << 2) | (x & 4) | ((x & 8) >> 2) | ((x & 16) >> 4);
}

// in-place 32-point DFT in registers: radix-2 decimation in frequency, natural-order input,
// v[p] = X[bitrev5(p)] on return.  Every index and twiddle is a compile-time constant after unrolling.
__device__ __forceinline__ void fft32(float2 (&v)[32]) {
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
#pragma unroll
    for (int g = 0; g < 32; g += 2 * half) {
#pragma unroll
      for (int j = 0; j < half; ++j) {
        const float2 a = v[g + j], b = v[g + j + half];
        v[g + j] = make_float2(a.x + b.x, a.y + b.y);
        const float2 d = make_float2(a.x - b.x, a.y - b.y);
        const int tk = j * (16 / half);            // W_{2 half}^j = W_32^{tk}
        if (tk == 0) v[g + j + half] = d;
        else if (tk == 8) v[g + j + half] = make_float2(d.y, -d.x);
        else v[g + j + half] = cmul(d, w32(tk));
      }
    }
  }
}

}  // namespace fftc
