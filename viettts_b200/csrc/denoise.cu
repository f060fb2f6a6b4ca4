// Bias denoiser of the vocoder output (the WaveGlow / HiFiGAN `Denoiser` convention), fp32 on the device in every
// vtts_precision mode:
//   STFT n_fft 1024 / hop 256 / periodic Hann, centered frames with reflect padding 512 (F = n / 256 + 1 frames, frame f
//   covers samples 256 f - 512 .. 256 f + 511) | |X| = sqrt(re^2 + im^2) | M' = max(|X| - s beta[k], 0) |
//   Y = X M' / |X| (0 where |X| = 0) | ISTFT: overlap-add of w * irfft(Y_f) over the envelope sum_f w^2.
// Rows of <= 512 samples cannot be reflect-padded and are copied.
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

#include "stft_common.cuh"
#include "vtts_internal.cuh"

namespace {

using fftc::bitrev5;
using stftc::fft1024;

constexpr int NF = vc::NFFT;      // 1024
constexpr int NB = vc::NBINS;     // 513
constexpr int HOP = vc::HOP;      // 256
constexpr int PAD = NF / 2;       // 512
constexpr int DN_WARPS = 4;       // frames per CTA
constexpr int TP = stftc::TP;     // transpose pitch (float2)
constexpr int OLA_THREADS = 256;
constexpr int DN_K = 2048;        // carried inputs per stream slot (the frames of a push start at most 1791 before P0)
constexpr int DN_LOOKAHEAD = 1023;

// rows == nullptr: the one-shot bounds of row b: n = n_in[b] clamped to [0, S] (or S), all S outputs written (zeros
// past n), frames 0 .. n / 256 when n > 512
__device__ __forceinline__ DnRow dn_row(const DnRow* rows, const int* n_in, int S, int b) {
  if (rows) return rows[b];
  DnRow r;
  r.n = n_in ? (long long)min(max(n_in[b], 0), S) : (long long)S;
  r.x0 = 0;
  r.g0 = 0;
  r.e0 = 0;
  r.cnt = S;
  r.copy = r.n <= PAD;
  r.nfr = r.copy ? 0 : (int)(r.n / HOP + 1);
  return r;
}

// MAG: write |X_0[k]| of frame 0 of row 0 to mag_out[k] (the bias of a waveform) and stop
template <bool MAG>
__global__ void __launch_bounds__(DN_WARPS * 32) denoise_frame_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                      const int* __restrict__ n_in, const DnRow* __restrict__ rows,
                                                                      const float* __restrict__ hann, const float2* __restrict__ tw,
                                                                      const float* __restrict__ bias, float strength,
                                                                      float* __restrict__ ws, int ws_frames, float* __restrict__ mag_out) {
  __shared__ float2 smem[DN_WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, fl = blockIdx.x * DN_WARPS + warp;
  const DnRow r = dn_row(rows, n_in, S, b);
  if (fl >= r.nfr || (MAG && fl > 0)) return;            // warps are independent: no block-level barrier below
  float2* sw = smem + (size_t)warp * 32 * TP;
  const float* xr = x + (size_t)b * x_ld;
  const long long g = r.g0 + fl;
  const long long j0 = g * HOP - PAD;

  // ---- windowed frame: sample j0 + lane + 32 m, reflected at 0 and n - 1 of the row ----
  float2 v[32];
  stftc::read_frame(v, xr, r.x0, r.n, j0, hann, lane);
  fft1024(v, sw, tw, lane);

  // ---- gain on bins k = lane + 32 k2 <= 512 ----
  __syncwarp();                                          // every lane has read sw
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k = lane + 32 * bitrev5(p);
    if (k <= NB - 1) {
      const float2 X = v[p];
      const float mag = sqrtf(X.x * X.x + X.y * X.y);
      if (MAG) {
        mag_out[k] = mag;
      } else {
        const float keep = fmaxf(mag - strength * __ldg(bias + k), 0.f);
        const float gain = mag > 0.f ? keep / mag : 0.f;
        sw[k] = make_float2(X.x * gain, X.y * gain);
      }
    }
  }
  if (MAG) return;
  __syncwarp();

  // ---- inverse: w * irfft(Y) of the gained spectrum ----
  stftc::inverse_frame(v, sw, tw, lane);
  stftc::write_frame(v, hann, lane, ws + ((size_t)b * ws_frames + fl) * NF);
}

__global__ void __launch_bounds__(OLA_THREADS) denoise_ola_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                  const int* __restrict__ n_in, const DnRow* __restrict__ rows,
                                                                  const float* __restrict__ hann, const float* __restrict__ ws,
                                                                  int ws_frames, float* __restrict__ y, long long y_ld) {
  const int b = blockIdx.y;
  const long long q = (long long)blockIdx.x * OLA_THREADS + threadIdx.x;
  const DnRow r = dn_row(rows, n_in, S, b);
  if (q >= r.cnt) return;
  const long long t = r.e0 + q;
  float out = 0.f;
  if (t < r.n) {
    if (r.copy) {
      out = x[(size_t)b * x_ld + (t - r.x0)];
    } else {
      // frames g with 256 g <= t + 512 <= 256 g + 1023 that exist (g <= n / 256), ascending
      const long long p = t + PAD;
      const long long g_lo = p >= NF - 1 ? (p - (NF - 1) + HOP - 1) / HOP : 0;
      const long long g_hi = min(r.n / HOP, p / HOP);
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

// frames then overlap-add: two launches
int dn_launch(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const DnRow* rows, int B, long long max_frames,
              long long max_out, float strength, const float* bias, float* ws, int ws_frames, float* y, long long y_ld, cudaStream_t st) {
  const float2* tw = reinterpret_cast<const float2*>(ctx->fft_tw);
  const unsigned fgrid = (unsigned)std::max(1LL, (max_frames + DN_WARPS - 1) / DN_WARPS);
  denoise_frame_kernel<false><<<dim3(fgrid, B), DN_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, ctx->hann, tw, bias, strength, ws, ws_frames,
                                                                      nullptr);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return vtts_denoise_ola(ctx, x, x_ld, S, n_in, rows, B, max_out, ws, ws_frames, y, y_ld, st);
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

int vtts_denoise_stream_lookahead(void) { return DN_LOOKAHEAD; }

int vtts_denoise(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, float strength, const float* bias_dev, float* y_dev,
                 void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!x_dev || !y_dev || !bias_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise: null pointer");
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise: y must not alias x");
  if (B < 1 || B > 65535 || S < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise: B=%d S=%d (1..65535, >= 1)", B, S);
  if (!finite_nonneg(strength)) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise: strength %g (finite and >= 0)", (double)strength);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const int ws_frames = S / HOP + 1;
  rc = ctx->ensure_ws((size_t)B * ws_frames * NF * sizeof(float));
  if (rc) return rc;
  return dn_launch(ctx, x_dev, S, S, n_dev, nullptr, B, ws_frames, S, strength, bias_dev, (float*)ctx->ws, ws_frames, y_dev, S,
                   (cudaStream_t)stream);
}

int vtts_denoise_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, float strength, const float* bias, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!x || !y || !bias || B < 1 || B > 65535 || S < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_host: bad argument (B=%d S=%d)", B, S);
  if (!finite_nonneg(strength)) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_host: strength %g (finite and >= 0)", (double)strength);
  int rc = dn_check_bias(ctx, "denoise_host", bias);
  if (rc) return rc;
  if (n_in)
    for (int b = 0; b < B; ++b)
      if (n_in[b] < 0 || n_in[b] > S) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_host: n[%d]=%d outside [0, %d]", b, n_in[b], S);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)B * S * 4, n_b = (size_t)B * 4, b_b = (size_t)NB * 4;
  const size_t o_n = (x_b + 255) & ~size_t(255), o_b = (o_n + n_b + 255) & ~size_t(255), o_y = (o_b + b_b + 255) & ~size_t(255);
  rc = ctx->ensure_staging(o_y + x_b, o_y + x_b);
  if (rc) return rc;
  char* hp = (char*)ctx->hpin;
  char* dp = (char*)ctx->dstage;
  cudaStream_t st = ctx->own_stream;
  memcpy(hp, x, x_b);
  if (n_in) memcpy(hp + o_n, n_in, n_b);
  memcpy(hp + o_b, bias, b_b);
  VTTS_CUDA(cudaMemcpyAsync(dp, hp, o_b + b_b, cudaMemcpyHostToDevice, st));
  rc = vtts_denoise(ctx, (const float*)dp, n_in ? (const int32_t*)(dp + o_n) : nullptr, B, S, strength, (const float*)(dp + o_b),
                    (float*)(dp + o_y), st);
  if (rc) {
    cudaStreamSynchronize(st);   // the staging copy must not outlive the call
    return rc;
  }
  VTTS_CUDA(cudaMemcpyAsync(hp + o_y, dp + o_y, x_b, cudaMemcpyDeviceToHost, st));
  VTTS_CUDA(cudaStreamSynchronize(st));
  memcpy(y, hp + o_y, x_b);
  return VTTS_OK;
}

int vtts_denoise_bias(vtts_ctx* ctx, const float* wav_dev, int n, float* bias_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!wav_dev || !bias_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_bias: null pointer");
  if (n <= PAD) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_bias: n=%d (more than %d samples)", n, PAD);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  denoise_frame_kernel<true><<<dim3(1, 1), DN_WARPS * 32, 0, (cudaStream_t)stream>>>(
      wav_dev, n, n, nullptr, nullptr, ctx->hann, reinterpret_cast<const float2*>(ctx->fft_tw), nullptr, 0.f, nullptr, 0, bias_dev);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct vtts_denoise_stream {
  vtts_ctx* ctx = nullptr;
  int S = 0, F = 0, cap = 0, out_pitch = 0, ws_frames = 0;
  float strength = 0.f;
  void* mem = nullptr;          // windows [S][cap], frame workspace [S][ws_frames][1024], bias [513], then the per-push tables
  float* win = nullptr;
  float* ws = nullptr;
  float* bias = nullptr;
  DnRow* d_rows = nullptr;
  int* d_prep = nullptr;
  // per slot: inputs received since BEGIN, outputs emitted, open, inputs of the last push whose tail has not moved yet
  std::vector<long long> P, E;
  std::vector<int> open, pending;
  std::vector<char> tbl;        // host image of the per-push tables: DnRow [S], then int [S][2]
};

int vtts_denoise_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, float strength, const float* bias,
                               vtts_denoise_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!out || !out_pitch || !bias) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_create: null pointer");
  *out = nullptr;
  if (max_streams < 1 || max_streams > 65535 || max_chunk_samples < 1 || max_chunk_samples > (1 << 22))
    return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_create: max_streams=%d max_chunk_samples=%d (1..65535, 1..%d)", max_streams,
                     max_chunk_samples, 1 << 22);
  if (!finite_nonneg(strength)) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_create: strength %g (finite and >= 0)", (double)strength);
  int rc = dn_check_bias(ctx, "denoise_stream_create", bias);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  vtts_denoise_stream* ds = new vtts_denoise_stream;
  ds->ctx = ctx;
  ds->S = max_streams;
  ds->F = max_chunk_samples;
  ds->cap = DN_K + max_chunk_samples;
  // outputs per push: fewer than n_new + 256 before END, at most n_new + 1023 with it (E(P0) >= P0 - 1023)
  ds->out_pitch = max_chunk_samples + DN_LOOKAHEAD;
  // frames per push: outputs [E0, E1) read frames floor((E0 - 511) / 256) .. floor((E1 + 511) / 256)
  ds->ws_frames = (ds->out_pitch + 2 * PAD) / HOP + 2;
  ds->strength = strength;
  const size_t win_b = ((size_t)max_streams * ds->cap * sizeof(float) + 255) & ~size_t(255);
  const size_t ws_b = (size_t)max_streams * ds->ws_frames * NF * sizeof(float);
  const size_t bias_b = ((size_t)NB * sizeof(float) + 255) & ~size_t(255);
  const size_t rows_b = ((size_t)max_streams * sizeof(DnRow) + 255) & ~size_t(255);
  const size_t bytes = win_b + ws_b + bias_b + rows_b + (size_t)max_streams * 2 * sizeof(int);
  cudaError_t e = cudaMalloc(&ds->mem, bytes);
  if (e == cudaSuccess) e = cudaMemset(ds->mem, 0, bytes);
  char* base = (char*)ds->mem;
  if (e == cudaSuccess) e = cudaMemcpy(base + win_b + ws_b, bias, (size_t)NB * sizeof(float), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (ds->mem) cudaFree(ds->mem);
    delete ds;
    return ctx->fail(e == cudaErrorMemoryAllocation ? VTTS_ERR_OOM : VTTS_ERR_CUDA, "denoise_stream_create: %zu bytes: %s", bytes,
                     cudaGetErrorString(e));
  }
  ds->win = (float*)base;
  ds->ws = (float*)(base + win_b);
  ds->bias = (float*)(base + win_b + ws_b);
  ds->d_rows = (DnRow*)(base + win_b + ws_b + bias_b);
  ds->d_prep = (int*)(base + win_b + ws_b + bias_b + rows_b);
  ds->P.assign(max_streams, 0);
  ds->E.assign(max_streams, 0);
  ds->open.assign(max_streams, 0);
  ds->pending.assign(max_streams, 0);
  ds->tbl.assign((size_t)max_streams * (sizeof(DnRow) + 2 * sizeof(int)), 0);
  *out = ds;
  *out_pitch = ds->out_pitch;
  return VTTS_OK;
}

int vtts_denoise_stream_destroy(vtts_ctx* ctx, vtts_denoise_stream* ds) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!ds) return VTTS_OK;
  if (ds->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_destroy: the stream belongs to another context");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());   // a push may still be running on the caller's stream
  cudaFree(ds->mem);
  delete ds;
  return VTTS_OK;
}

int vtts_denoise_stream_push(vtts_ctx* ctx, vtts_denoise_stream* ds, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                             float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!ds || ds->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push: the stream belongs to another context");
  if (!x_dev || !n_new || !flags || !y_dev || !n_out) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push: null pointer");
  const int S = ds->S, F = ds->F;
  for (int s = 0; s < S; ++s) {
    if (n_new[s] < 0 || n_new[s] > F) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push: n_new[%d]=%d outside [0, %d]", s, n_new[s], F);
    if (flags[s] & ~3u) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push: flags[%d]=%u (bit0 BEGIN, bit1 END)", s, flags[s]);
    const bool idle = n_new[s] == 0 && flags[s] == 0;
    if (!idle && !(flags[s] & 1) && !ds->open[s])
      return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push: slot %d is not open (push BEGIN first, also after END)", s);
  }
  VTTS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;

  // ---- host bookkeeping: outputs [E0, E1) of this push and the frames they read ----
  DnRow* rows = reinterpret_cast<DnRow*>(ds->tbl.data());
  int* prep = reinterpret_cast<int*>(ds->tbl.data() + (size_t)S * sizeof(DnRow));
  std::vector<long long> E1(S);
  long long max_out = 0, max_frames = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = n_new[s] > 0 || flags[s] != 0, begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : ds->P[s], E0 = begin ? 0 : ds->E[s], P1 = P0 + n_new[s];
    long long e = E0;
    if (act) e = end ? P1 : std::min(P1, (long long)HOP * std::max(0LL, P1 / HOP - 3));
    E1[s] = e;
    n_out[s] = (int32_t)(e - E0);
    DnRow r{};
    r.x0 = P0 - DN_K;
    r.n = end ? P1 : DN_OPEN;
    r.e0 = E0;
    r.cnt = e - E0;
    r.copy = end && P1 <= PAD;
    if (r.cnt > 0 && !r.copy) {
      const long long p0 = E0 + PAD, p1 = e - 1 + PAD;
      r.g0 = p0 >= NF - 1 ? (p0 - (NF - 1) + HOP - 1) / HOP : 0;
      r.nfr = (int)(std::min(r.n / HOP, p1 / HOP) - r.g0 + 1);
    }
    if (r.nfr > ds->ws_frames || r.cnt > ds->out_pitch)
      return ctx->fail(VTTS_ERR_CUDA, "denoise_stream_push: slot %d needs %d frames / %lld outputs (internal bound %d / %d)", s, r.nfr,
                       r.cnt, ds->ws_frames, ds->out_pitch);
    rows[s] = r;
    prep[2 * s] = act && !begin ? ds->pending[s] : 0;
    prep[2 * s + 1] = act ? n_new[s] : 0;
    max_out = std::max(max_out, r.cnt);
    max_frames = std::max(max_frames, (long long)r.nfr);
  }

  // ---- device: table copies, prep, frames, overlap-add (three launches) ----
  // pageable source: the call returns once the table is staged, so ds->tbl may be rewritten by the next push
  VTTS_CUDA(cudaMemcpyAsync(ds->d_rows, rows, (size_t)S * sizeof(DnRow), cudaMemcpyHostToDevice, st));
  VTTS_CUDA(cudaMemcpyAsync(ds->d_prep, prep, (size_t)S * 2 * sizeof(int), cudaMemcpyHostToDevice, st));
  int rc = vtts_stream_window_prep(ctx, ds->win, ds->cap, DN_K, ds->d_prep, x_dev, F, S, st);
  if (rc) return rc;
  rc = dn_launch(ctx, ds->win, ds->cap, ds->cap, nullptr, ds->d_rows, S, max_frames, max_out, ds->strength, ds->bias, ds->ws, ds->ws_frames,
                 y_dev, ds->out_pitch, st);
  if (rc) return rc;

  // ---- commit the slot state ----
  for (int s = 0; s < S; ++s) {
    const bool act = n_new[s] > 0 || flags[s] != 0, begin = flags[s] & 1, end = flags[s] & 2;
    if (!act) continue;
    ds->P[s] = (begin ? 0 : ds->P[s]) + n_new[s];
    ds->E[s] = E1[s];
    ds->open[s] = !end;
    ds->pending[s] = end ? 0 : n_new[s];
  }
  return VTTS_OK;
}

int vtts_denoise_stream_push_host(vtts_ctx* ctx, vtts_denoise_stream* ds, const float* x, const int32_t* n_new, const uint8_t* flags,
                                  float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!ds || ds->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push_host: the stream belongs to another context");
  if (!x || !y) return ctx->fail(VTTS_ERR_BAD_ARG, "denoise_stream_push_host: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)ds->S * ds->F * 4, y_b = (size_t)ds->S * ds->out_pitch * 4;
  const size_t o_y = (x_b + 255) & ~size_t(255);
  int rc = ctx->ensure_staging(o_y + y_b, o_y + y_b);
  if (rc) return rc;
  char* hp = (char*)ctx->hpin;
  char* dp = (char*)ctx->dstage;
  cudaStream_t st = ctx->own_stream;
  memcpy(hp, x, x_b);
  VTTS_CUDA(cudaMemcpyAsync(dp, hp, x_b, cudaMemcpyHostToDevice, st));
  rc = vtts_denoise_stream_push(ctx, ds, (const float*)dp, n_new, flags, (float*)(dp + o_y), n_out, st);
  if (rc) {
    cudaStreamSynchronize(st);   // the staging copy must not outlive the call
    return rc;
  }
  VTTS_CUDA(cudaMemcpyAsync(hp + o_y, dp + o_y, y_b, cudaMemcpyDeviceToHost, st));
  VTTS_CUDA(cudaStreamSynchronize(st));
  memcpy(y, hp + o_y, y_b);
  return VTTS_OK;
}
