// Bias denoiser of the vocoder output (the WaveGlow / HiFiGAN `Denoiser` convention), fp32 on the device in every
// vtts_precision mode:
//   STFT n_fft 1024 / hop 256 / periodic Hann, centered frames with reflect padding 512 (F = n / 256 + 1 frames, frame f
//   covers samples 256 f - 512 .. 256 f + 511) | |X| = sqrt(re^2 + im^2) | M' = max(|X| - s beta[k], 0) |
//   Y = X M' / |X| (0 where |X| = 0) | ISTFT: overlap-add of w * irfft(Y_f) over the envelope sum_f w^2.
// Rows of <= 512 samples cannot be reflect-padded and are copied.  The frame kernel (with the gain below as its policy)
// and the stream's schedule are stft_gain.cuh's, shared with the watermark embedder (watermark.cu).
//
// Frame kernel.  One warp per frame.  The frame is transformed ALONE: a complex FFT-1024 of the windowed real frame
// (imaginary part zero), four-step 32 x 32 with both 32-point passes in registers (fftc::fft32) and exact table
// twiddles between them; the gain is applied to bins 0..512; the inverse is the same forward transform of the
// conjugated, Hermitian-completed spectrum (Re FFT(conj Y) = N * irfft(Y); the imaginary parts of bins 0 and 512 drop
// out as irfft drops them), times 1 / 1024 and the window.  A frame's output bits are therefore a function of its own
// 1024 input samples, the strength and the bias -- MelFilter's packing of two frames into one complex FFT would mix a
// frame's bins with its partner's, which a stream may not have received yet.  The price is a transform twice the
// size of a real-input one; at two FFT-1024s per 256 samples that is immaterial next to the generator.
//
// Overlap-add kernel.  One thread per output: the covering frames in ascending order, numerator and envelope in fp32,
// one division.  An output depends on its index and the frames' bits only, so any schedule that computes the same
// frames produces the same bits: the stream recomputes the (up to three) frames an earlier push already used instead
// of carrying partial sums.
//
// Stream.  Per slot a window of K = 2048 carried inputs plus one chunk (the prep step of the resample stream moves the
// tail); an output t is emitted once the frames covering it are final, i.e. after 256 floor(t / 256) + 1024 inputs:
// before END a slot that has received P samples has emitted min(P, 256 max(0, floor(P / 256) - 3)).
#include <algorithm>
#include <cmath>
#include <cstring>

#include "stft_gain.cuh"

namespace {

using stftg::HOP;
using stftg::NB;
using stftg::NF;
using stftg::PAD;
constexpr int OLA_THREADS = 256;

// spectral subtraction: |X| less strength * bias[k], floored at 0, with X's phase
struct DnGain {
  const float* __restrict__ bias;
  float strength;
  __device__ __forceinline__ float2 operator()(int k, long long, float2 X) const {
    const float mag = sqrtf(X.x * X.x + X.y * X.y);
    const float keep = fmaxf(mag - strength * __ldg(bias + k), 0.f);
    const float gain = mag > 0.f ? keep / mag : 0.f;
    return make_float2(X.x * gain, X.y * gain);
  }
};

// |X_0[k]| of frame 0 of a row of n > 512 samples into mag_out[k] (the bias of a waveform); one warp
__global__ void __launch_bounds__(32) denoise_mag_kernel(const float* __restrict__ x, long long n, const float* __restrict__ hann,
                                                         const float2* __restrict__ tw, float* __restrict__ mag_out) {
  __shared__ float2 sw[32 * stftc::TP];
  const int lane = threadIdx.x;
  float2 v[32];
  stftc::read_frame(v, x, 0, n, -PAD, hann, lane);
  stftc::fft1024(v, sw, tw, lane);
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k = lane + 32 * fftc::bitrev5(p);
    if (k <= NB - 1) mag_out[k] = sqrtf(v[p].x * v[p].x + v[p].y * v[p].y);
  }
}

__global__ void __launch_bounds__(OLA_THREADS) denoise_ola_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                  const int* __restrict__ n_in, const DnRow* __restrict__ rows,
                                                                  const float* __restrict__ hann, const float* __restrict__ ws,
                                                                  int ws_frames, float* __restrict__ y, long long y_ld) {
  const int b = blockIdx.y;
  const long long q = (long long)blockIdx.x * OLA_THREADS + threadIdx.x;
  const DnRow r = stftg::frame_row(rows, n_in, S, b);
  if (q >= r.cnt) return;
  const long long t = r.e0 + q;
  float out = 0.f;
  if (t < r.n) {
    if (r.copy) {
      out = x[(size_t)b * x_ld + (t - r.x0)];
    } else {
      // frames g with 256 g < t + 512 <= 256 g + 1023 that exist (g <= n / 256), ascending.  A frame's sample 0 is
      // windowed by w[0] = 0 and adds exactly nothing, so it is not read: a stream may release an output before the
      // frame that starts at it is synthesized.
      const long long p = t + PAD;
      const long long g_lo = p >= NF - 1 ? (p - (NF - 1) + HOP - 1) / HOP : 0;
      const long long g_hi = min(r.n / HOP, (p - 1) / HOP);
      const float* wr = ws + (size_t)b * ws_frames * NF;
      float num = 0.f, env = 0.f;
      for (long long g = g_lo; g <= g_hi; ++g) {
        const int o = (int)(p - g * HOP);
        const float h = __ldg(hann + o);
        num += wr[(size_t)(g - r.g0) * NF + o];
        env = fmaf(h, h, env);
      }
      out = num / env;
    }
  }
  y[(size_t)b * y_ld + q] = out;
}

bool finite_nonneg(float v) { return std::isfinite(v) && v >= 0.f; }

int dn_check_bias(vtts_ctx* ctx, const char* who, const float* bias) {
  for (int k = 0; k < NB; ++k)
    if (!finite_nonneg(bias[k])) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: bias[%d] = %g (finite and >= 0)", who, k, (double)bias[k]);
  return VTTS_OK;
}

}  // namespace

int vtts_denoise_ola(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const DnRow* rows, int B, long long max_out,
                     const float* ws, int ws_frames, float* y, long long y_ld, cudaStream_t st) {
  const unsigned ogrid = (unsigned)std::max(1LL, (max_out + OLA_THREADS - 1) / OLA_THREADS);
  denoise_ola_kernel<<<dim3(ogrid, B), OLA_THREADS, 0, st>>>(x, x_ld, S, n_in, rows, ctx->hann, ws, ws_frames, y, y_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

int vtts_denoise_stream_lookahead(void) { return stftg::LOOKAHEAD; }

namespace {

// the parameters and batch shape of a one-shot call of entry point `who`
int dn_args(vtts_ctx* ctx, const char* who, int B, int S, float strength) {
  const int rc = batch_check(ctx, who, B, S, S_ANY);
  if (rc) return rc;
  if (!finite_nonneg(strength)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: strength %g (finite and >= 0)", who, (double)strength);
  return VTTS_OK;
}

int dn_launch(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, float strength, const float* bias, float* y, cudaStream_t st) {
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const int ws_frames = S / HOP + 1;
  rc = ctx->ensure_ws((size_t)B * ws_frames * NF * sizeof(float));
  if (rc) return rc;
  return stftg::launch(ctx, x, S, S, n_in, nullptr, B, ws_frames, S, DnGain{bias, strength}, (float*)ctx->ws, ws_frames, y, S, st);
}

}  // namespace

int vtts_denoise(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, float strength, const float* bias_dev, float* y_dev,
                 void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = dn_args(ctx, "denoise", B, S, strength);
  if (rc) return rc;
  if (!x_dev || !y_dev || !bias_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise: null pointer");
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise: y must not alias x");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return dn_launch(ctx, x_dev, n_dev, B, S, strength, bias_dev, y_dev, (cudaStream_t)stream);
}

int vtts_denoise_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, float strength, const float* bias, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = dn_args(ctx, "denoise_host", B, S, strength);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("denoise_host", x, n_in, B, S, y && bias);
  if (!rc) rc = dn_check_bias(ctx, "denoise_host", bias);
  if (rc) return rc;
  const size_t o_b = hs.in(bias, (size_t)NB * 4), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return dn_launch(ctx, hs.x(), hs.n(), B, S, strength, hs.dev<const float>(o_b), hs.dev<float>(o_y), st); });
}

int vtts_denoise_bias(vtts_ctx* ctx, const float* wav_dev, int n, float* bias_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!wav_dev || !bias_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_bias: null pointer");
  if (n <= PAD) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_bias: n=%d (more than %d samples)", n, PAD);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  denoise_mag_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(wav_dev, n, ctx->hann, reinterpret_cast<const float2*>(ctx->fft_tw), bias_dev);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct vtts_denoise_stream : stftg::Stream {
  using Stream::Stream;
  float strength = 0.f;
  float* bias = nullptr;        // [513]
};

int vtts_denoise_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, float strength, const float* bias,
                               vtts_denoise_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "denoise_stream_create", out, out_pitch && bias, max_streams, max_chunk_samples);
  if (rc) return rc;
  if (!finite_nonneg(strength)) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_create: strength %g (finite and >= 0)", (double)strength);
  rc = dn_check_bias(ctx, "denoise_stream_create", bias);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  std::unique_ptr<vtts_denoise_stream> ds(new vtts_denoise_stream(ctx, max_streams, max_chunk_samples));
  ds->strength = strength;
  rc = stream_alloc(ctx, "denoise_stream_create", *ds, [&](Arena& a) {
    ds->carve_window(a);
    ds->carve_ws(a);
    ds->bias = a.take<float>(NB);
    ds->carve_tables(a);
  });
  if (rc) return rc;
  VTTS_CUDA(cudaMemcpy(ds->bias, bias, (size_t)NB * sizeof(float), cudaMemcpyHostToDevice));
  *out_pitch = ds->out_pitch;
  *out = ds.release();
  return VTTS_OK;
}

int vtts_denoise_stream_destroy(vtts_ctx* ctx, vtts_denoise_stream* ds) { return stream_destroy(ctx, "denoise_stream_destroy", ds); }

int vtts_denoise_stream_push(vtts_ctx* ctx, vtts_denoise_stream* ds, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                             float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "denoise_stream_push", ds, x_dev && n_new && flags && y_dev && n_out);
  if (!rc) rc = ds->slots.check(ctx, "denoise_stream_push", ds->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return ds->push("denoise_stream_push", x_dev, n_new, flags, y_dev, n_out, DnGain{ds->bias, ds->strength}, false, (cudaStream_t)stream);
}

int vtts_denoise_stream_push_host(vtts_ctx* ctx, vtts_denoise_stream* ds, const float* x, const int32_t* n_new, const uint8_t* flags,
                                  float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "denoise_stream_push_host", ds, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ds->S * ds->F * 4), o_y = hs.out((size_t)ds->S * ds->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return vtts_denoise_stream_push(ctx, ds, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, st);
  });
}
