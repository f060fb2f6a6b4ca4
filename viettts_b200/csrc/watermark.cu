// Keyed spread-spectrum watermark of synthesized speech, fp32 on the device in every vtts_precision mode
// (oracle/watermark_oracle.py is the float64 definition).
//
// Embed (16 kHz, key kappa = (lo, hi), strength eps): the denoiser's STFT (stft_gain.cuh: n_fft 1024, hop 256, periodic
// Hann, centered frames with reflect padding) with the gain Y_f[k] = X_f[k] (1 + eps c(kappa, j, k)) on the band
// k in [20, 219) (312..3422 Hz), every other bin unchanged, j = floor(f / 4) mod 64; then the denoiser's overlap-add.
// c(kappa, j, k) = +1, or -1 when the top bit of word 0 of threefry2x32(lo, hi, j, k) is set.  The chip pattern repeats
// every 64 groups of 4 frames: 65536 samples.  eps = 0 copies the rows bit for bit, as rows of <= 512 samples are copied.
//
// Detect: resample to 16 kHz when the rate differs (vtts_resample), then
//   spec: one warp per hop-64 frame t (the same centered framing), D_t[k] = M[k] - (sum_{|i| <= 4} M[k + i]) / 9 on the
//         band, M = log(|X|^2 + 1e-12): the log power whitened by its 9-bin moving mean across frequency;
//   fold: per frame phase q (hop-256 frames f at t = q + 4 f) the group sums G_g = sum_{i < 4} D_{q + 16 g + 4 i}, the
//         neighbour-subtracted H_g = G_g - (G_{g-1} + G_{g+1}) / 2 (0 for the first and the last group) and the fold
//         S_q[j] = sum_{g = j mod 64} H_g, ascending g;
//   corr: per row and key, z(p, q) = sum_{j,k} S_q[j][k] c(kappa, (j + p) mod 64, k) / sqrt(sum S_q^2) (0 when that is 0),
//         as the 64 x 64 product A = S_q C^T over k followed by the circular diagonal sums z(p) = sum_j A[j][(j + p) mod 64].
// Aligned mode reads p = q = 0.  Search mode keeps the largest z over the 1024 (p, q) and reports its offset
// (1024 p - 64 q) mod 65536: where the row's sample 0 sits in the mark's period, so a crop that started at sample c of a
// marked row reports c mod 65536 (c a multiple of 64).  Every sum has one fixed order, so a row's z and offset are the same
// alone and at any batch position.
#include <algorithm>
#include <cmath>
#include <numeric>

#include "stft_gain.cuh"
#include "threefry.cuh"

namespace {

using stftg::NF;
using stftg::PAD;

constexpr int WM_K0 = 20, WM_K1 = 219, WM_NK = WM_K1 - WM_K0;   // band bins
constexpr int WM_G = 4;                 // hop-256 frames per chip group
constexpr int WM_P = 64;                // groups per period
constexpr int WM_Q = 16;                // frame phases of the search (hop 64 within one group of 1024 samples)
constexpr int DET_HOP = 64;
constexpr int DET_RATE = 16000;
constexpr int WM_PERIOD = WM_P * WM_G * stftg::HOP;   // 65536 samples
constexpr float WM_MAX_STRENGTH = 0.3f;
constexpr int WM_MAX_KEYS = 4096;
constexpr int SPEC_WARPS = 4;
constexpr int FOLD_THREADS = 224;       // >= WM_NK
constexpr int CORR_THREADS = 256;       // a 4 x 4 tile of A = S C^T per thread
constexpr int CORR_SMEM = 2 * WM_NK * WM_P * (int)sizeof(float);

__device__ __forceinline__ bool chip_neg(uint32_t k0, uint32_t k1, uint32_t j, uint32_t k) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, j, k, o0, o1);
  return (o0 >> 31) != 0;
}

struct WmGain {
  uint32_t k0, k1;
  float up, dn;    // 1 + eps, 1 - eps
  __device__ __forceinline__ float2 operator()(int k, long long f, float2 X) const {
    if (k < WM_K0 || k >= WM_K1) return X;
    const float g = chip_neg(k0, k1, (uint32_t)((f / WM_G) % WM_P), (uint32_t)k) ? dn : up;
    return make_float2(X.x * g, X.y * g);
  }
};

WmGain wm_gain(uint64_t key, float eps) { return WmGain{(uint32_t)key, (uint32_t)(key >> 32), 1.f + eps, 1.f - eps}; }

// eps = 0: y = x on [0, n), 0 past n
__global__ void wm_copy_kernel(const float* __restrict__ x, const int* __restrict__ n_in, int S, float* __restrict__ y) {
  const int b = blockIdx.y;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S) return;
  const int n = n_in ? min(max(n_in[b], 0), S) : S;
  y[(size_t)b * S + t] = t < n ? x[(size_t)b * S + t] : 0.f;
}

// row b's length at 16 kHz: n_in[b] (clamped to [0, S], or S) resampled by up / down, as vtts_resample writes it
__device__ __forceinline__ long long det_len(const int* n_in, int S, int b, int up, int down) {
  const long long n = n_in ? min(max(n_in[b], 0), S) : S;
  return (n * up + down - 1) / down;
}
__device__ __forceinline__ int det_frames(long long n16) { return n16 > PAD ? (int)(n16 / DET_HOP + 1) : 0; }

// D [B][T_ld][199]: the whitened band of every hop-64 frame
__global__ void __launch_bounds__(SPEC_WARPS * 32) wm_spec_kernel(const float* __restrict__ x, long long x_ld, const int* __restrict__ n_in,
                                                                  int S, int up, int down, const float* __restrict__ hann,
                                                                  const float2* __restrict__ tw, float* __restrict__ D, int T_ld) {
  __shared__ float2 smem[SPEC_WARPS * 32 * stftc::TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, t = blockIdx.x * SPEC_WARPS + warp;
  const long long n = det_len(n_in, S, b, up, down);
  if (t >= det_frames(n)) return;                        // warps are independent: no block-level barrier below
  float2* sw = smem + (size_t)warp * 32 * stftc::TP;
  float2 v[32];
  stftc::read_frame(v, x + (size_t)b * x_ld, 0, n, (long long)t * DET_HOP - PAD, hann, lane);
  stftc::fft1024(v, sw, tw, lane);
  __syncwarp();                                          // every lane has read sw
  float* M = reinterpret_cast<float*>(sw);               // M[k - 16] for k in [16, 224)
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k = lane + 32 * fftc::bitrev5(p);
    if (k >= WM_K0 - 4 && k < WM_K1 + 5) M[k - (WM_K0 - 4)] = logf(fmaf(v[p].x, v[p].x, v[p].y * v[p].y) + 1e-12f);
  }
  __syncwarp();
  float* out = D + ((size_t)b * T_ld + t) * WM_NK;
  for (int i = lane; i < WM_NK; i += 32) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < 9; ++d) s += M[i + d];
    out[i] = M[i + 4] - s * (1.f / 9.f);
  }
}

// S [B][nq][64][199]: the group / neighbour / period fold of phase q; grid (64, nq, B)
__global__ void __launch_bounds__(FOLD_THREADS) wm_fold_kernel(const float* __restrict__ D, int T_ld, const int* __restrict__ n_in, int S,
                                                               int up, int down, float* __restrict__ Sf) {
  const int j = blockIdx.x, q = blockIdx.y, nq = gridDim.y, b = blockIdx.z, k = threadIdx.x;
  if (k >= WM_NK) return;
  const int T = det_frames(det_len(n_in, S, b, up, down));
  const int Fq = T > q ? (T - 1 - q) / 4 + 1 : 0;
  const int ng = Fq / WM_G;
  const float* Db = D + (size_t)b * T_ld * WM_NK + k;
  auto gsum = [&](int g) {
    const float* d = Db + (size_t)(q + 16 * g) * WM_NK;
    return ((d[0] + d[4 * WM_NK]) + d[8 * WM_NK]) + d[12 * WM_NK];
  };
  float acc = 0.f;
  for (int g = j; g < ng - 1; g += WM_P)
    if (g > 0) acc += gsum(g) - 0.5f * (gsum(g - 1) + gsum(g + 1));
  Sf[(((size_t)b * nq + q) * WM_P + j) * WM_NK + k] = acc;
}

// z [B][K], offset [B][K]; grid (K, B).  Shared: chips C[k][m] = +-1 of the block's key, then per phase the fold
// S[k][j]; A [64][65] reuses S's space once the product is done.
__global__ void __launch_bounds__(CORR_THREADS) wm_corr_kernel(const float* __restrict__ Sf, int nq, int np, const uint64_t* __restrict__ keys,
                                                               float* __restrict__ z_out, int* __restrict__ off_out) {
  extern __shared__ float sm[];
  float* Cs = sm;                       // [199][64]
  float* Ss = sm + WM_NK * WM_P;        // [199][64], then A [64][65]
  __shared__ float red[CORR_THREADS];
  __shared__ float zbest[WM_P];
  __shared__ int obest[WM_P];
  const int key = blockIdx.x, b = blockIdx.y, K = gridDim.x, tid = threadIdx.x;
  const uint64_t kv = keys[key];
  const uint32_t k0 = (uint32_t)kv, k1 = (uint32_t)(kv >> 32);
  for (int i = tid; i < WM_NK * WM_P; i += CORR_THREADS) {
    const int k = i / WM_P, m = i % WM_P;
    Cs[i] = chip_neg(k0, k1, (uint32_t)m, (uint32_t)(k + WM_K0)) ? -1.f : 1.f;
  }
  const int jt = tid & 15, mt = tid >> 4;   // rows 4 jt .. 4 jt + 3 of A, columns 4 mt .. 4 mt + 3
  float best = -INFINITY;
  int best_off = 0;
  for (int q = 0; q < nq; ++q) {
    __syncthreads();                      // the previous phase is done with Ss (and the chips are in on the first)
    const float* src = Sf + ((size_t)b * nq + q) * WM_P * WM_NK;
    float ss = 0.f;
    for (int i = tid; i < WM_NK * WM_P; i += CORR_THREADS) {
      const int j = i / WM_NK, k = i % WM_NK;
      const float s = src[i];
      Ss[k * WM_P + j] = s;
      ss = fmaf(s, s, ss);
    }
    red[tid] = ss;
    __syncthreads();
    for (int w = CORR_THREADS / 2; w > 0; w >>= 1) {
      if (tid < w) red[tid] += red[tid + w];
      __syncthreads();
    }
    const float norm = sqrtf(red[0]);
    float acc[4][4] = {};
    for (int k = 0; k < WM_NK; ++k) {
      const float4 s = *reinterpret_cast<const float4*>(Ss + k * WM_P + 4 * jt);
      const float4 c = *reinterpret_cast<const float4*>(Cs + k * WM_P + 4 * mt);
      const float sv[4] = {s.x, s.y, s.z, s.w}, cv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[a][e] = fmaf(sv[a], cv[e], acc[a][e]);
    }
    __syncthreads();                      // every thread is done reading Ss
    float* A = Ss;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int e = 0; e < 4; ++e) A[(4 * jt + a) * (WM_P + 1) + 4 * mt + e] = acc[a][e];
    __syncthreads();
    if (tid < np) {
      const int p = tid;
      float zs = 0.f;
      for (int j = 0; j < WM_P; ++j) zs += A[j * (WM_P + 1) + ((j + p) & (WM_P - 1))];
      const float zv = norm > 0.f ? zs / norm : 0.f;
      const int off = ((1024 * p - DET_HOP * q) % WM_PERIOD + WM_PERIOD) % WM_PERIOD;
      if (zv > best || (zv == best && off < best_off)) {
        best = zv;
        best_off = off;
      }
    }
  }
  // the largest z over the phases p this block's threads kept, the smallest offset among equal ones
  if (tid < WM_P) {
    zbest[tid] = tid < np ? best : -INFINITY;
    obest[tid] = best_off;
  }
  __syncthreads();
  if (tid == 0) {
    float bz = zbest[0];
    int bo = obest[0];
    for (int p = 1; p < np; ++p)
      if (zbest[p] > bz || (zbest[p] == bz && obest[p] < bo)) {
        bz = zbest[p];
        bo = obest[p];
      }
    z_out[(size_t)b * K + key] = bz;
    off_out[(size_t)b * K + key] = bo;
  }
}

int wm_check_strength(vtts_ctx* ctx, const char* who, float eps) {
  if (!(eps >= 0.f && eps <= WM_MAX_STRENGTH))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: strength %g (in [0, %g])", who, (double)eps, (double)WM_MAX_STRENGTH);
  return VTTS_OK;
}

// a row of S samples at `rate` resampled to the detector's rate
long long det_samples(int S, int rate) {
  const long long g = std::gcd(rate, DET_RATE);
  return ((long long)S * (DET_RATE / g) + rate / g - 1) / (rate / g);
}

// the parameters and batch shape of a watermark call of entry point `who`
int wm_args(vtts_ctx* ctx, const char* who, int B, int S, float strength) {
  const int rc = batch_check(ctx, who, B, S, S_ANY);
  return rc ? rc : wm_check_strength(ctx, who, strength);
}

int wm_launch(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, uint64_t key, float strength, float* y, cudaStream_t st) {
  if (strength == 0.f) {
    wm_copy_kernel<<<dim3((unsigned)((S + 255) / 256), B), 256, 0, st>>>(x, n_in, S, y);
    ctx->launches++;
    VTTS_CUDA(cudaGetLastError());
    return VTTS_OK;
  }
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const int ws_frames = S / stftg::HOP + 1;
  rc = ctx->ensure_ws((size_t)B * ws_frames * NF * sizeof(float));
  if (rc) return rc;
  return stftg::launch(ctx, x, S, S, n_in, nullptr, B, ws_frames, S, wm_gain(key, strength), (float*)ctx->ws, ws_frames, y, S, st);
}

// ... and of a detect call; the row at the detector's rate must stay within 2^30 samples
int det_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, int K) {
  const int rc = batch_check(ctx, who, B, S, S_ANY);
  if (rc) return rc;
  if (K < 1 || K > WM_MAX_KEYS) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: K=%d keys (1..%d)", who, K, WM_MAX_KEYS);
  if (rate < 8000 || rate > 192000 || vtts_resample_filter(rate, DET_RATE, nullptr, 0) < 0)
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rate %d (8000..192000, a ratio to 16000 the resampler takes)", who, rate);
  if (det_samples(S, rate) > (1LL << 30)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: S=%d at %d Hz is too long", who, S, rate);
  return VTTS_OK;
}

int det_launch(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const uint64_t* keys, int K, int search, float* z,
               int32_t* offset, cudaStream_t st) {
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const long long g = std::gcd(rate, DET_RATE);
  const int up = (int)(DET_RATE / g), down = (int)(rate / g);
  const long long S16 = det_samples(S, rate);
  const int T_ld = (int)(S16 / DET_HOP + 1), nq = search ? WM_Q : 1, np = search ? WM_P : 1;
  Arena m(nullptr, 0, true);
  auto carve = [&](Arena& a, float** x16, float** D, float** Sf) {
    *x16 = up == down ? nullptr : a.take<float>((size_t)B * S16);
    *D = a.take<float>((size_t)B * T_ld * WM_NK);
    *Sf = a.take<float>((size_t)B * nq * WM_P * WM_NK);
  };
  float *x16, *D, *Sf;
  carve(m, &x16, &D, &Sf);
  rc = ctx->ensure_ws(m.off);
  if (rc) return rc;
  Arena a((char*)ctx->ws, ctx->ws_bytes, false);
  carve(a, &x16, &D, &Sf);
  const float* src = x;
  if (x16) {
    rc = vtts_resample_run(ctx, rate, DET_RATE, x, S, S, n_in, nullptr, B, S16, S16, x16, S16, st);
    if (rc) return rc;
    src = x16;
  }
  wm_spec_kernel<<<dim3((unsigned)((T_ld + SPEC_WARPS - 1) / SPEC_WARPS), B), SPEC_WARPS * 32, 0, st>>>(
      src, x16 ? S16 : S, n_in, S, up, down, ctx->hann, reinterpret_cast<const float2*>(ctx->fft_tw), D, T_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  wm_fold_kernel<<<dim3(WM_P, nq, B), FOLD_THREADS, 0, st>>>(D, T_ld, n_in, S, up, down, Sf);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  VTTS_CUDA(cudaFuncSetAttribute(wm_corr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CORR_SMEM));
  wm_corr_kernel<<<dim3(K, B), CORR_THREADS, CORR_SMEM, st>>>(Sf, nq, np, keys, z, offset);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace

int vtts_watermark_stream_lookahead(void) { return stftg::LOOKAHEAD; }

int vtts_watermark(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, uint64_t key, float strength, float* y_dev,
                   void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = wm_args(ctx, "watermark", B, S, strength);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "watermark: null pointer");
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "watermark: y must not alias x");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return wm_launch(ctx, x_dev, n_dev, B, S, key, strength, y_dev, (cudaStream_t)stream);
}

int vtts_watermark_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, uint64_t key, float strength, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = wm_args(ctx, "watermark_host", B, S, strength);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("watermark_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return wm_launch(ctx, hs.x(), hs.n(), B, S, key, strength, hs.dev<float>(o_y), st); });
}

int vtts_watermark_detect(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, const uint64_t* keys_dev, int K,
                          int search, float* z_dev, int32_t* offset_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = det_args(ctx, "watermark_detect", B, S, rate, K);
  if (rc) return rc;
  if (!x_dev || !keys_dev || !z_dev || !offset_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "watermark_detect: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return det_launch(ctx, x_dev, n_dev, B, S, rate, keys_dev, K, search, z_dev, offset_dev, (cudaStream_t)stream);
}

int vtts_watermark_detect_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const uint64_t* keys, int K,
                               int search, float* z, int32_t* offset) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = det_args(ctx, "watermark_detect_host", B, S, rate, K);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("watermark_detect_host", x, n_in, B, S, keys && z && offset);
  if (rc) return rc;
  const size_t out_b = (size_t)B * K * 4, o_k = hs.in(keys, (size_t)K * 8), o_z = hs.out(out_b, z), o_o = hs.out(out_b, offset);
  return hs.run([&](cudaStream_t st) {
    return det_launch(ctx, hs.x(), hs.n(), B, S, rate, hs.dev<const uint64_t>(o_k), K, search, hs.dev<float>(o_z), hs.dev<int32_t>(o_o), st);
  });
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct vtts_watermark_stream : stftg::Stream {
  using Stream::Stream;
  uint64_t key = 0;
  float strength = 0.f;
};

int vtts_watermark_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, uint64_t key, float strength,
                                 vtts_watermark_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "watermark_stream_create", out, out_pitch != nullptr, max_streams, max_chunk_samples);
  if (rc) return rc;
  rc = wm_check_strength(ctx, "watermark_stream_create", strength);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  std::unique_ptr<vtts_watermark_stream> ws(new vtts_watermark_stream(ctx, max_streams, max_chunk_samples));
  ws->key = key;
  ws->strength = strength;
  rc = stream_alloc(ctx, "watermark_stream_create", *ws, [&](Arena& a) {
    ws->carve_window(a);
    ws->carve_ws(a);
    ws->carve_tables(a);
  });
  if (rc) return rc;
  *out_pitch = ws->out_pitch;
  *out = ws.release();
  return VTTS_OK;
}

int vtts_watermark_stream_destroy(vtts_ctx* ctx, vtts_watermark_stream* ws) { return stream_destroy(ctx, "watermark_stream_destroy", ws); }

int vtts_watermark_stream_push(vtts_ctx* ctx, vtts_watermark_stream* ws, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                               float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "watermark_stream_push", ws, x_dev && n_new && flags && y_dev && n_out);
  if (!rc) rc = ws->slots.check(ctx, "watermark_stream_push", ws->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return ws->push("watermark_stream_push", x_dev, n_new, flags, y_dev, n_out, wm_gain(ws->key, ws->strength), ws->strength == 0.f,
                  (cudaStream_t)stream);
}

int vtts_watermark_stream_push_host(vtts_ctx* ctx, vtts_watermark_stream* ws, const float* x, const int32_t* n_new, const uint8_t* flags,
                                    float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "watermark_stream_push_host", ws, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ws->S * ws->F * 4), o_y = hs.out((size_t)ws->S * ws->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return vtts_watermark_stream_push(ctx, ws, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, st);
  });
}
