// Warp-level STFT frame code shared by the bias denoiser (denoise.cu) and the pitch shifter (pitch.cu): the windowed
// read of one centered frame with reflection, the forward four-step FFT-1024 and the inverse of a half spectrum.
// One warp owns one frame; lane `lane` holds samples lane + 32 m in v[m].  Each frame is transformed alone, so its bits
// depend on its own 1024 input samples only.
#pragma once

#include <cuda_runtime.h>

#include "fft_common.cuh"

namespace stftc {

constexpr int NF = 1024;     // n_fft
constexpr int NB = 513;      // bins 0..512
constexpr int TP = 33;       // transpose pitch (float2) of a warp's 32 x TP buffer

// windowed frame starting at absolute sample j0: v[m] = x[j] * hann[lane + 32 m], j = j0 + lane + 32 m reflected at 0 and
// n - 1 of the row; xr holds the row with absolute sample x0 at element 0
__device__ __forceinline__ void read_frame(float2 (&v)[32], const float* __restrict__ xr, long long x0, long long n, long long j0,
                                           const float* __restrict__ hann, int lane) {
  if (j0 >= 0 && j0 + NF <= n) {
    const float* src = xr + (j0 - x0) + lane;
#pragma unroll
    for (int m = 0; m < 32; ++m) v[m] = make_float2(__ldg(src + 32 * m) * __ldg(hann + lane + 32 * m), 0.f);
  } else {
#pragma unroll
    for (int m = 0; m < 32; ++m) {
      long long j = j0 + lane + 32 * m;
      j = j < 0 ? -j : (j >= n ? 2 * (n - 1) - j : j);
      v[m] = make_float2(__ldg(xr + (j - x0)) * __ldg(hann + lane + 32 * m), 0.f);
    }
  }
}

// forward four-step FFT-1024 of v (v[m] = sample lane + 32 m): on return v[p] = X[lane + 32 bitrev5(p)].  sw is the
// warp's 32 x TP transpose buffer; the caller syncs the warp before sw is reused.
__device__ __forceinline__ void fft1024(float2 (&v)[32], float2* sw, const float2* __restrict__ tw, int lane) {
  fftc::fft32(v);                                        // over m: v[bitrev5(k1)] = sum_m x[lane + 32 m] W32^(m k1)
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k1 = fftc::bitrev5(p);
    sw[k1 * TP + lane] = k1 == 0 ? v[p] : fftc::cmul(v[p], __ldg(tw + lane * k1));   // W1024^(lane k1), lane k1 <= 961
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < 32; ++t) v[t] = sw[lane * TP + t];  // lane = k1, t = the first pass's lane
  fftc::fft32(v);                                        // over t: X[k1 + 32 k2]
}

// inverse of the half spectrum Y[0..512] held in sw[0..512] (written by the whole warp, synced): Re FFT(conj Y) of the
// Hermitian completion = 1024 irfft(Y), the imaginary parts of bins 0 and 512 dropping out as irfft drops them; on return
// v[p].x = 1024 irfft(Y)[lane + 32 bitrev5(p)] (write_frame stores it)
__device__ __forceinline__ void inverse_frame(float2 (&v)[32], float2* sw, const float2* __restrict__ tw, int lane) {
  // element i = lane + 32 m is conj Y[i] (i <= 512) or Y[1024 - i]
#pragma unroll
  for (int m = 0; m < 32; ++m) {
    const int i = lane + 32 * m;
    if (m < 16 || i == NB - 1) {
      const float2 y = sw[i];
      v[m] = make_float2(y.x, -y.y);
    } else {
      v[m] = sw[NF - i];
    }
  }
  __syncwarp();                                          // every lane has read the spectrum
  fft1024(v, sw, tw, lane);
}

// out[i] = w[i] * irfft(Y)[i] from inverse_frame's v
__device__ __forceinline__ void write_frame(const float2 (&v)[32], const float* __restrict__ hann, int lane, float* out) {
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int i = lane + 32 * fftc::bitrev5(p);
    out[i] = v[p].x * (1.f / NF) * __ldg(hann + i);
  }
}

}  // namespace stftc
