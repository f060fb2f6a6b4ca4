// STFT + log-mel -- restates MelFilter.__call__ (vietTTS/nat/dsp.py:115-128):
//   reflect pad 384 | frame 1024 / hop 256 | periodic Hann | FFT-1024, bins 0..512 |
//   sqrt(re^2+im^2+1e-9) | 80x513 Slaney filterbank | log(max(.,1e-5))
// One WARP per pair of frames, no block-level barrier anywhere.  The two real frames are packed into one complex
// FFT-1024 (frame A real part, frame B imaginary part) and separated afterwards.  The FFT is the four-step
// factorisation 1024 = 32 x 32 with both 32-point transforms held entirely in registers (radix-2 DIF, twiddles
// folded to immediates), so data crosses shared memory exactly once between the two passes (padded pitch 33:
// conflict free both ways) instead of once per radix-4 pass.  Frame B's samples are frame A's shifted by the hop:
// 40 coalesced 128 B loads per lane column serve both frames; the 4x overlap between pairs is served by L1/L2, so
// every sample is read from HBM once.
#include <math.h>

#include "fft_common.cuh"
#include "vtts_internal.cuh"

namespace {

using fftc::bitrev5;
using fftc::cmul;
using fftc::fft32;

constexpr int NF = vc::NFFT;      // 1024
constexpr int NB = vc::NBINS;     // 513
constexpr int MEL_WARPS = 8;      // frame pairs per CTA
constexpr int TP = 33;            // transpose pitch (float2)

// sqrt.approx.f32: one MUFU op, max relative error 2^-23 (the IEEE sqrtf expands to ~10 instructions; 34 of them per
// lane were a quarter of the kernel)
__device__ __forceinline__ float fast_sqrt(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__global__ void __launch_bounds__(MEL_WARPS * 32) melspec_kernel(const float* __restrict__ wav, int S, int F,
                                                                 const float* __restrict__ hann, const float2* __restrict__ tw,
                                                                 const float* __restrict__ fb, const int* __restrict__ lo,
                                                                 const int* __restrict__ hi, float* __restrict__ mel) {
  extern __shared__ __align__(16) float2 smem2[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, pair = blockIdx.x * MEL_WARPS + warp;
  const int fa = pair * 2, fbn = fa + 1;
  if (fa >= F) return;                              // warps are independent: no block-level barrier below
  const bool hasB = fbn < F;
  float2* sw = smem2 + (size_t)warp * 32 * TP;
  const float* y = wav + (size_t)b * S;

  // ---- samples n = lane + 32 m of frame A (m < 32) and of frame B (= A shifted by 256 samples = 8 m-steps) ----
  float2 v[32];
  {
    float raw[40];
    const int base = fa * vc::HOP - 384 + lane;     // reflect pad p = 384 (dsp.py:119-121)
    if (fa * vc::HOP >= 384 && fa * vc::HOP + 896 <= S) {   // whole 1280-sample window interior (warp uniform): no index math
#pragma unroll
      for (int m = 0; m < 40; ++m) raw[m] = __ldg(y + base + 32 * m);
    } else {
#pragma unroll
      for (int m = 0; m < 40; ++m) {
        int i = base + 32 * m;
        i = i < 0 ? -i : (i >= S ? 2 * (S - 1) - i : i);
        raw[m] = (m < 32 || hasB) ? __ldg(y + i) : 0.f;
      }
    }
#pragma unroll
    for (int m = 0; m < 32; ++m) {
      const float h = __ldg(hann + lane + 32 * m);
      v[m] = make_float2(raw[m] * h, raw[m + 8] * h);
    }
  }
  // ---- pass 1: DFT over m, then the inter-pass twiddle exp(-2 pi i lane k1 / 1024), k1 = 0..31 ----
  fft32(v);
  {
    const float2 w1 = __ldg(tw + lane);
    const float2 w2 = cmul(w1, w1), w3 = cmul(w2, w1), w4 = cmul(w2, w2);
    float2 r[4] = {make_float2(1.f, 0.f), w1, w2, w3};   // four interleaved power chains: r[c] = w1^(4 q + c)
#pragma unroll
    for (int q = 0; q < 8; ++q) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int k1 = 4 * q + c;
        const float2 x = v[bitrev5(k1)];
        sw[k1 * TP + lane] = k1 == 0 ? x : cmul(x, r[c]);
        if (q < 7) r[c] = cmul(r[c], w4);
      }
    }
  }
  __syncwarp();
  // ---- pass 2: lane = k1, DFT over t: X[k1 + 32 k2] ----
#pragma unroll
  for (int t = 0; t < 32; ++t) v[t] = sw[lane * TP + t];
  fft32(v);
  __syncwarp();
#pragma unroll
  for (int p = 0; p < 32; ++p) sw[lane + 32 * bitrev5(p)] = v[p];          // Z[k], k = k1 + 32 k2, linear
  __syncwarp();
  // ---- separate the two real transforms, magnitude (dsp.py:124-125) ----
  // Z = FFT(a + i b):  A[k] = (Z[k] + conj(Z[N-k]))/2,  B[k] = (Z[k] - conj(Z[N-k]))/(2i)
  float mA[17], mB[17];
#pragma unroll
  for (int j = 0; j < 17; ++j) {
    const int k = lane + 32 * j;
    mA[j] = mB[j] = 0.f;
    if (k < NB) {
      const float2 z = sw[k];
      const float2 zc = sw[(NF - k) & (NF - 1)];
      const float ar = 0.5f * (z.x + zc.x), ai = 0.5f * (z.y - zc.y);
      const float br = 0.5f * (z.y + zc.y), bi = -0.5f * (z.x - zc.x);
      mA[j] = fast_sqrt(ar * ar + ai * ai + 1e-9f);
      mB[j] = fast_sqrt(br * br + bi * bi + 1e-9f);
    }
  }
  __syncwarp();
  float* magA = reinterpret_cast<float*>(sw);
  float* magB = magA + 520;
#pragma unroll
  for (int j = 0; j < 17; ++j) {
    const int k = lane + 32 * j;
    if (k < NB) { magA[k] = mA[j]; magB[k] = mB[j]; }
  }
  __syncwarp();
  // ---- filterbank (only the non-zero span of each triangle) + log (dsp.py:126-127) ----
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int m = lane + 32 * q;
    if (m < vc::MEL) {
      const float* frow = fb + (size_t)m * NB;
      float sa = 0.f, sb = 0.f;
      const int k1 = hi[m];
      for (int k = lo[m]; k < k1; ++k) {
        const float w = __ldg(frow + k);
        sa = fmaf(w, magA[k], sa);
        sb = fmaf(w, magB[k], sb);
      }
      mel[((size_t)b * F + fa) * vc::MEL + m] = logf(fmaxf(sa, 1e-5f));
      if (hasB) mel[((size_t)b * F + fbn) * vc::MEL + m] = logf(fmaxf(sb, 1e-5f));
    }
  }
}

__global__ void mel_span_kernel(const float* __restrict__ fb, int* lo, int* hi) {
  const int m = threadIdx.x;
  if (m >= vc::MEL) return;
  int l = NB, h = 0;
  for (int k = 0; k < NB; ++k)
    if (fb[(size_t)m * NB + k] != 0.f) {
      if (k < l) l = k;
      h = k + 1;
    }
  if (h == 0) l = 0;
  lo[m] = l;
  hi[m] = h;
}

}  // namespace

int vtts_fft_tables(vtts_ctx* ctx) {
  if (ctx->fft_ready) return VTTS_OK;
  // twiddles exp(-2 pi i k / 1024) and the periodic Hann window, computed in double on the host
  std::vector<float> tw(2 * NF), hn(NF);
  for (int k = 0; k < NF; ++k) {
    const double a = -2.0 * M_PI * (double)k / (double)NF;
    tw[2 * k] = (float)cos(a);
    tw[2 * k + 1] = (float)sin(a);
    hn[k] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)k / (double)NF));  // np.hanning(1025)[:-1], dsp.py:81
  }
  if (!ctx->fft_tw) VTTS_CUDA(cudaMalloc(&ctx->fft_tw, tw.size() * sizeof(float)));
  if (!ctx->hann) VTTS_CUDA(cudaMalloc(&ctx->hann, hn.size() * sizeof(float)));
  VTTS_CUDA(cudaMemcpy(ctx->fft_tw, tw.data(), tw.size() * sizeof(float), cudaMemcpyHostToDevice));
  VTTS_CUDA(cudaMemcpy(ctx->hann, hn.data(), hn.size() * sizeof(float), cudaMemcpyHostToDevice));
  ctx->fft_ready = true;
  return VTTS_OK;
}

int vtts_melspec_prepare(vtts_ctx* ctx) {
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  if (!ctx->mel_lo) VTTS_CUDA(cudaMalloc(&ctx->mel_lo, vc::MEL * sizeof(int)));
  if (!ctx->mel_hi) VTTS_CUDA(cudaMalloc(&ctx->mel_hi, vc::MEL * sizeof(int)));
  mel_span_kernel<<<1, 128>>>(ctx->mel_fb, ctx->mel_lo, ctx->mel_hi);
  VTTS_CUDA(cudaGetLastError());
  VTTS_CUDA(cudaDeviceSynchronize());
  VTTS_CUDA(cudaFuncSetAttribute(melspec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MEL_WARPS * 32 * TP * (int)sizeof(float2)));
  return VTTS_OK;
}

int vtts_melspec_run(vtts_ctx* ctx, const float* wav, int B, int S, float* mel, cudaStream_t st) {
  if (!ctx->mel_loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "mel filterbank not loaded");
  if (B < 1 || B > 65535 || S < 512 || S % vc::HOP != 0)
    return ctx->fail(VTTS_ERR_BAD_ARG, "melspec: B=%d S=%d (need S %% 256 == 0, S >= 512)", B, S);
  const int F = S / vc::HOP;
  const int pairs = (F + 1) / 2;
  dim3 grid((pairs + MEL_WARPS - 1) / MEL_WARPS, B);
  constexpr size_t smem = (size_t)MEL_WARPS * 32 * TP * sizeof(float2);
  melspec_kernel<<<grid, MEL_WARPS * 32, smem, st>>>(wav, S, F, ctx->hann, reinterpret_cast<const float2*>(ctx->fft_tw), ctx->mel_fb,
                                       ctx->mel_lo, ctx->mel_hi, mel);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}
