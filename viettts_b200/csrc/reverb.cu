// Convolution reverb: a uniformly partitioned overlap-save FIR, fp32 on the device in every vtts_precision mode.
//   c[t] = sum_{i <= min(t, L - 1)} h[i] x[t - i]  (causal, zero state);  y[t] = (1 - mix) x[t] + mix c[t] for t < n, 0 past n.
//
// Block grid.  Blocks and partitions are 512 samples, transforms 1024.  H_k = FFT([h[512k .. 512k + 511], 0 x 512]) for
// k < K = ceil(L / 512); X_j = FFT(x over [512 (j - 1), 512 (j + 1))), zeros before 0 and from n on; output block j (samples
// 512 j .. 512 j + 511) is samples 512..1023 of irfft(sum_{k <= min(j, K - 1)} X_{j-k} H_k).  Each spectrum is 513 bins.
//
// Bits.  Every X_j and H_k is the stftc FFT-1024 of its own 1024 samples, one warp each.  Each bin's sum runs over k in
// ascending order with one fixed fp32 expression (four fmaf), whatever the tiling, and the inverse of a block reads
// only that block's sum, so a row gives the same bits alone, at any batch position and through the stream.
//
// Launches.  A one-shot call is four: IR partitions -> H, input frames -> X, the multiply-accumulate into the block
// spectra, inverse and mix.  The MAC kernel gives each warp 32 bins x JG = 16 consecutive output blocks of one row:
// lane = bin, one accumulator per block.  Block u of the group needs X_{ja + u - k} at step k, so the warp keeps the 16
// spectra X_{ja - k} .. X_{ja - k + 15} in a register ring and loads one new X and one H_k per step for 16 complex
// multiply-adds: every X element loaded serves 16 output blocks.
//
// Stream.  Per slot a window of 1023 carried inputs plus one chunk (vtts_stream_window_prep) and a ring of the slot's
// last R input spectra; block j is released once its frame is complete (P >= 512 (j + 1)), END releases the rest.
#include <algorithm>
#include <cmath>
#include <memory>

#include "stft_common.cuh"
#include "stream_common.cuh"

namespace {

using fftc::bitrev5;

constexpr int NF = stftc::NF;          // 1024
constexpr int NB = stftc::NB;          // 513
constexpr int TP = stftc::TP;
constexpr int BLK = 512;               // block and partition size
constexpr int FR_WARPS = 4;            // frames per CTA of the transform kernels
constexpr int JG = 16;                 // output blocks per warp of the MAC
constexpr int MAC_WARPS = 8;           // block groups per CTA of the MAC (the same 32 bins: H_k is shared through L1)
constexpr int BIN_TILES = (NB + 31) / 32;
constexpr int RV_K = 2 * BLK - 1;      // carried inputs per stream slot
constexpr int RV_LOOKAHEAD = BLK - 1;

// where a row's buffers sit in absolute time, and what a launch computes of it
struct RvRow {
  long long x0;     // absolute index of input buffer element 0
  long long n;      // inputs at or past n read as zero (the row's length, or what a stream slot has received)
  long long j0;     // first output block; outputs are written from sample 512 j0 on
  long long cnt;    // outputs written
  int nblk;         // output blocks computed (blocks j0 .. j0 + nblk - 1); later written outputs are zero
  int pad;
};

// rows == nullptr: the one-shot bounds of row b (n_in[b] clamped to [0, S], or S; all S outputs written)
__device__ __forceinline__ RvRow rv_row(const RvRow* rows, const int* n_in, int S, int b) {
  if (rows) return rows[b];
  RvRow r;
  r.n = n_in ? (long long)min(max(n_in[b], 0), S) : (long long)S;
  r.x0 = 0;
  r.j0 = 0;
  r.cnt = S;
  r.nblk = (int)((r.n + BLK - 1) / BLK);
  r.pad = 0;
  return r;
}

// unwindowed frame starting at absolute sample j0: v[m] = x[j], j = j0 + lane + 32 m, for j in [lo, hi), else 0; xr holds
// absolute sample x0 at element 0
__device__ __forceinline__ void read_block(float2 (&v)[32], const float* __restrict__ xr, long long x0, long long lo, long long hi,
                                           long long j0, int lane) {
#pragma unroll
  for (int m = 0; m < 32; ++m) {
    const long long j = j0 + lane + 32 * m;
    v[m] = make_float2(j >= lo && j < hi ? __ldg(xr + (j - x0)) : 0.f, 0.f);
  }
}

// bins 0..512 of fft1024's v to out[0..512]
__device__ __forceinline__ void write_bins(const float2 (&v)[32], int lane, float2* __restrict__ out) {
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k = lane + 32 * bitrev5(p);
    if (k < NB) out[k] = v[p];
  }
}

// H_k for k < K, one warp each: H [K][513]
__global__ void __launch_bounds__(FR_WARPS * 32) reverb_ir_kernel(const float* __restrict__ h, int L, int K, const float2* __restrict__ tw,
                                                                  float2* __restrict__ H) {
  __shared__ float2 smem[FR_WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = blockIdx.x * FR_WARPS + warp;
  if (k >= K) return;
  float2 v[32];
  const long long lo = (long long)k * BLK;
  read_block(v, h, 0, lo, min((long long)L, lo + BLK), lo, lane);
  stftc::fft1024(v, smem + (size_t)warp * 32 * TP, tw, lane);
  write_bins(v, lane, H + (size_t)k * NB);
}

// X_j of output blocks j0 .. j0 + nblk - 1 of each row, one warp each, into the row's ring X [B][R][513] at j mod R
__global__ void __launch_bounds__(FR_WARPS * 32) reverb_frame_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                     const int* __restrict__ n_in, const RvRow* __restrict__ rows,
                                                                     const float2* __restrict__ tw, float2* __restrict__ X, int R) {
  __shared__ float2 smem[FR_WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, jl = blockIdx.x * FR_WARPS + warp;
  const RvRow r = rv_row(rows, n_in, S, b);
  if (jl >= r.nblk) return;
  const long long j = r.j0 + jl;
  float2 v[32];
  read_block(v, x + (size_t)b * x_ld, r.x0, 0, r.n, (j - 1) * BLK, lane);
  stftc::fft1024(v, smem + (size_t)warp * 32 * TP, tw, lane);
  write_bins(v, lane, X + ((size_t)b * R + (size_t)(j % R)) * NB);
}

__device__ __forceinline__ void cmac(float2& acc, float2 x, float2 h) {
  acc.x = fmaf(x.x, h.x, acc.x);
  acc.x = fmaf(-x.y, h.y, acc.x);
  acc.y = fmaf(x.x, h.y, acc.y);
  acc.y = fmaf(x.y, h.x, acc.y);
}

// one step k of a block group (ja: its first block; t = k mod 16): win[(u - t) & 15] holds X_{ja + u - k}.  GUARD: the
// step may lie past kmax, and block u takes it only when k <= ja + u (the sum of block j stops at k = j)
template <bool GUARD>
__device__ __forceinline__ void mac_step(float2 (&acc)[JG], float2 (&win)[JG], int t, int k, long long ja, int kmax, int& ring, int R,
                                         const float2* __restrict__ Xr, const float2* __restrict__ Hb) {
  if (GUARD && k > kmax) return;
  if (k > 0) {
    ring = ring == 0 ? R - 1 : ring - 1;                 // ring index of X_{ja - k}
    if (!GUARD || ja - k >= 0) win[(JG - t) & (JG - 1)] = __ldg(Xr + (size_t)ring * NB);
  }
  const float2 hk = __ldg(Hb + (size_t)k * NB);
#pragma unroll
  for (int u = 0; u < JG; ++u)
    if (!GUARD || k <= ja + u) cmac(acc[u], win[(u - t) & (JG - 1)], hk);
}

// Y [B][ycap][513]: block spectrum j0 + jl at row jl, for jl < nblk
__global__ void __launch_bounds__(MAC_WARPS * 32, 2) reverb_mac_kernel(const float2* __restrict__ X, int R, const float2* __restrict__ H,
                                                                       int K, int S, const int* __restrict__ n_in,
                                                                       const RvRow* __restrict__ rows, float2* __restrict__ Y, int ycap) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.z, bin = blockIdx.x * 32 + lane;
  const RvRow r = rv_row(rows, n_in, S, b);
  const int jl0 = (blockIdx.y * MAC_WARPS + warp) * JG;
  if (jl0 >= r.nblk) return;                             // warps are independent: no block-level barrier below
  const long long ja = r.j0 + jl0;
  const float2* Xr = X + (size_t)b * R * NB + min(bin, NB - 1);
  const float2* Hb = H + min(bin, NB - 1);
  // blocks past nblk are computed from whatever their ring rows hold and never stored
  int ring = (int)(ja % R);
  float2 acc[JG], win[JG];
#pragma unroll
  for (int u = 0; u < JG; ++u) {
    const int i = ring + u;
    win[u] = __ldg(Xr + (size_t)(i >= R ? i - R : i) * NB);
    acc[u] = make_float2(0.f, 0.f);
  }
  const int kmax = (int)min(ja + JG - 1, (long long)K - 1);   // the last step any block of the group takes
  const long long kall = min(ja, (long long)K - 1);           // every block takes steps 0 .. kall
  int k0 = 0;
  for (; k0 + JG - 1 <= kall; k0 += JG) {
#pragma unroll
    for (int t = 0; t < JG; ++t) mac_step<false>(acc, win, t, k0 + t, ja, kmax, ring, R, Xr, Hb);
  }
  for (; k0 <= kmax; k0 += JG) {
#pragma unroll
    for (int t = 0; t < JG; ++t) mac_step<true>(acc, win, t, k0 + t, ja, kmax, ring, R, Xr, Hb);
  }
  if (bin >= NB) return;
  float2* yb = Y + ((size_t)b * ycap + jl0) * NB + bin;
#pragma unroll
  for (int u = 0; u < JG; ++u)
    if (jl0 + u < r.nblk) yb[(size_t)u * NB] = acc[u];
}

// outputs: block jl of a row is samples 512..1023 of irfft(Y row jl), mixed with the dry input; y [B][y_ld] from sample
// 512 j0 on, cnt outputs, 0 at or past n
__global__ void __launch_bounds__(FR_WARPS * 32) reverb_out_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                   const int* __restrict__ n_in, const RvRow* __restrict__ rows,
                                                                   const float2* __restrict__ tw, const float2* __restrict__ Y, int ycap,
                                                                   float dry, float wet, float* __restrict__ y, long long y_ld) {
  __shared__ float2 smem[FR_WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, jl = blockIdx.x * FR_WARPS + warp;
  const RvRow r = rv_row(rows, n_in, S, b);
  const long long q0 = (long long)jl * BLK;              // the block's first output
  if (q0 >= r.cnt) return;
  float* yr = y + (size_t)b * y_ld;
  if (jl >= r.nblk) {                                    // past the row's last block
    for (int i = lane; i < BLK; i += 32)
      if (q0 + i < r.cnt) yr[q0 + i] = 0.f;
    return;
  }
  float2* sw = smem + (size_t)warp * 32 * TP;
  const float2* Yb = Y + ((size_t)b * ycap + jl) * NB;
  for (int k = lane; k < NB; k += 32) sw[k] = Yb[k];
  __syncwarp();
  float2 v[32];
  stftc::inverse_frame(v, sw, tw, lane);
  const long long t0 = (r.j0 + jl) * BLK;
  const float* xb = x + (size_t)b * x_ld + (t0 - r.x0);
  float* yb = yr + q0;
  const int n_w = (int)min(r.cnt - q0, (long long)BLK), n_x = (int)max(0LL, min(r.n - t0, (long long)BLK));
#pragma unroll
  for (int p = 1; p < 32; p += 2) {                      // bitrev5(p) >= 16: samples 512..1023, the overlap-save half
    const int i = lane + 32 * bitrev5(p) - BLK;
    if (i >= n_w) continue;
    float out = 0.f;
    if (i < n_x) {
      const float xv = xb[i];
      out = wet == 0.f ? xv : fmaf(wet, v[p].x * (1.f / NF), dry * xv);
    }
    yb[i] = out;
  }
}

int partitions(int L) { return (L + BLK - 1) / BLK; }

int rv_check(vtts_ctx* ctx, const char* who, int rate, int L, float mix) {
  if (rate < 8000 || rate > 192000) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rate %d (8000..192000)", who, rate);
  if (L < 1 || (long long)L > 5LL * rate) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: L=%d taps (1..5 rate = %lld)", who, L, 5LL * rate);
  if (!(mix >= 0.f && mix <= 1.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: mix %g (in [0, 1])", who, (double)mix);
  return VTTS_OK;
}

int rv_check_ir(vtts_ctx* ctx, const char* who, const float* ir, int L) {
  for (int i = 0; i < L; ++i)
    if (!std::isfinite(ir[i])) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: ir[%d] = %g (finite)", who, i, (double)ir[i]);
  return VTTS_OK;
}

int rv_ir(vtts_ctx* ctx, const float* ir, int L, float2* H, cudaStream_t st) {
  const int K = partitions(L);
  reverb_ir_kernel<<<(K + FR_WARPS - 1) / FR_WARPS, FR_WARPS * 32, 0, st>>>(ir, L, K, reinterpret_cast<const float2*>(ctx->fft_tw), H);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// frames, MAC, inverse and mix: three launches.  max_blk: the most blocks a row computes; max_cnt: the most outputs
int rv_launch(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const RvRow* rows, int B, long long max_blk,
              long long max_cnt, const float2* H, int K, float2* X, int R, float2* Y, int ycap, float mix, float* y, long long y_ld,
              cudaStream_t st) {
  const float2* tw = reinterpret_cast<const float2*>(ctx->fft_tw);
  const unsigned fgrid = (unsigned)std::max(1LL, (max_blk + FR_WARPS - 1) / FR_WARPS);
  reverb_frame_kernel<<<dim3(fgrid, B), FR_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, tw, X, R);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  const unsigned mgrid = (unsigned)std::max(1LL, (max_blk + JG * MAC_WARPS - 1) / (JG * MAC_WARPS));
  reverb_mac_kernel<<<dim3(BIN_TILES, mgrid, B), MAC_WARPS * 32, 0, st>>>(X, R, H, K, S, n_in, rows, Y, ycap);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  const unsigned ogrid = (unsigned)std::max(1LL, ((max_cnt + BLK - 1) / BLK + FR_WARPS - 1) / FR_WARPS);
  reverb_out_kernel<<<dim3(ogrid, B), FR_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, tw, Y, ycap, 1.f - mix, mix, y, y_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// the parameters and batch shape of a one-shot call of entry point `who`
int rv_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, int L, float mix) {
  const int rc = batch_check(ctx, who, B, S, S_ANY);
  return rc ? rc : rv_check(ctx, who, rate, L, mix);
}

int rv_oneshot(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* ir, int L, float mix, float* y, cudaStream_t st) {
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const int K = partitions(L);
  const long long nbS = ((long long)S + BLK - 1) / BLK;
  const int R = (int)nbS + JG, ycap = (int)nbS;          // X rows past a row's blocks only feed blocks that are not stored
  Arena m(nullptr, 0, true);
  const auto carve = [&](Arena& a, float2** H, float2** X, float2** Y) {
    *H = a.take<float2>((size_t)K * NB);
    *X = a.take<float2>((size_t)B * R * NB);
    *Y = a.take<float2>((size_t)B * ycap * NB);
  };
  float2 *H, *X, *Y;
  carve(m, &H, &X, &Y);
  rc = ctx->ensure_ws(m.off);
  if (rc) return rc;
  Arena a(ctx->ws, m.off, false);
  carve(a, &H, &X, &Y);
  rc = rv_ir(ctx, ir, L, H, st);
  if (rc) return rc;
  return rv_launch(ctx, x, S, S, n_in, nullptr, B, nbS, S, H, K, X, R, Y, ycap, mix, y, S, st);
}

}  // namespace

int vtts_reverb_stream_lookahead(void) { return RV_LOOKAHEAD; }

int vtts_reverb(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, const float* ir_dev, int L, float mix,
                float* y_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = rv_args(ctx, "reverb", B, S, rate, L, mix);
  if (rc) return rc;
  if (!x_dev || !y_dev || !ir_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "reverb: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return rv_oneshot(ctx, x_dev, n_dev, B, S, ir_dev, L, mix, y_dev, (cudaStream_t)stream);
}

int vtts_reverb_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const float* ir, int L, float mix, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = rv_args(ctx, "reverb_host", B, S, rate, L, mix);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("reverb_host", x, n_in, B, S, y && ir);
  if (!rc) rc = rv_check_ir(ctx, "reverb_host", ir, L);
  if (rc) return rc;
  const size_t o_h = hs.in(ir, (size_t)L * 4), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return rv_oneshot(ctx, hs.x(), hs.n(), B, S, hs.dev<const float>(o_h), L, mix, hs.dev<float>(o_y), st); });
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct vtts_reverb_stream : SampleStream<RvRow> {
  using SampleStream::SampleStream;
  int out_pitch = 0, K = 0, R = 0, ycap = 0;
  float mix = 0.f;
  float2* H = nullptr;          // [K][513], computed at create
  float2* X = nullptr;          // per slot the ring of its last R input spectra [S][R][513]
  float2* Y = nullptr;          // block spectra of a push [S][ycap][513]
  float* ir = nullptr;          // [L], the IR as given
};

int vtts_reverb_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, const float* ir, int L, float mix,
                              vtts_reverb_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "reverb_stream_create", out, out_pitch && ir, max_streams, max_chunk_samples);
  if (rc) return rc;
  rc = rv_check(ctx, "reverb_stream_create", rate, L, mix);
  if (!rc) rc = rv_check_ir(ctx, "reverb_stream_create", ir, L);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  std::unique_ptr<vtts_reverb_stream> rs(new vtts_reverb_stream(ctx, max_streams, max_chunk_samples, RV_K));
  rs->out_pitch = max_chunk_samples + RV_LOOKAHEAD;
  rs->K = partitions(L);
  // blocks per push: at most ceil((511 + F) / 512) (a slot holds at most 511 unreleased inputs); the ring keeps the
  // K - 1 spectra before a push's first block and the push's own
  rs->ycap = (max_chunk_samples + 2 * BLK - 2) / BLK;
  rs->R = rs->K + rs->ycap - 1;
  rs->mix = mix;
  rc = stream_alloc(ctx, "reverb_stream_create", *rs, [&](Arena& a) {
    rs->carve_window(a);
    rs->H = a.take<float2>((size_t)rs->K * NB);
    rs->X = a.take<float2>((size_t)max_streams * rs->R * NB);
    rs->Y = a.take<float2>((size_t)max_streams * rs->ycap * NB);
    rs->ir = a.take<float>(L);
    rs->carve_tables(a);
  });
  if (rc) return rc;
  VTTS_CUDA(cudaMemcpy(rs->ir, ir, (size_t)L * sizeof(float), cudaMemcpyHostToDevice));
  rc = rv_ir(ctx, rs->ir, L, rs->H, ctx->own_stream);
  if (rc) return rc;
  VTTS_CUDA(cudaStreamSynchronize(ctx->own_stream));
  *out_pitch = rs->out_pitch;
  *out = rs.release();
  return VTTS_OK;
}

int vtts_reverb_stream_destroy(vtts_ctx* ctx, vtts_reverb_stream* rs) { return stream_destroy(ctx, "reverb_stream_destroy", rs); }

int vtts_reverb_stream_push(vtts_ctx* ctx, vtts_reverb_stream* rs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                            float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "reverb_stream_push", rs, x_dev && n_new && flags && y_dev && n_out);
  if (!rc) rc = rs->slots.check(ctx, "reverb_stream_push", rs->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = rs->S;
  const SlotState& sl = rs->slots;

  // ---- host bookkeeping: outputs [E0, E1) of this push, blocks E0 / 512 .. ceil(E1 / 512) - 1 ----
  RvRow* rows = rs->rows<0>();
  std::vector<long long> E1(S);
  long long max_cnt = 0, max_blk = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : sl.P[s], E0 = begin ? 0 : sl.E[s], P1 = P0 + n_new[s];
    long long e = E0;
    if (act) e = end ? P1 : BLK * (P1 / BLK);
    E1[s] = e;
    n_out[s] = (int32_t)(e - E0);
    RvRow r{};
    r.x0 = P0 - RV_K;
    r.n = P1;
    r.j0 = E0 / BLK;
    r.cnt = e - E0;
    r.nblk = (int)((e + BLK - 1) / BLK - r.j0);
    if (r.nblk > rs->ycap || r.cnt > rs->out_pitch)
      return ctx->fail(VTTS_ERR_CUDA, "reverb_stream_push: slot %d needs %d blocks / %lld outputs (internal bound %d / %d)", s, r.nblk,
                       r.cnt, rs->ycap, rs->out_pitch);
    rows[s] = r;
    max_cnt = std::max(max_cnt, r.cnt);
    max_blk = std::max(max_blk, (long long)r.nblk);
  }

  // ---- device: one table copy, window step, frames, MAC, inverse and mix (four launches) ----
  rc = rs->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  rc = rv_launch(ctx, rs->win, rs->cap, rs->cap, nullptr, rs->d_rows<0>(), S, max_blk, max_cnt, rs->H, rs->K, rs->X, rs->R, rs->Y,
                 rs->ycap, rs->mix, y_dev, rs->out_pitch, st);
  if (rc) return rc;
  rs->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_reverb_stream_push_host(vtts_ctx* ctx, vtts_reverb_stream* rs, const float* x, const int32_t* n_new, const uint8_t* flags, float* y,
                                 int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "reverb_stream_push_host", rs, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)rs->S * rs->F * 4), o_y = hs.out((size_t)rs->S * rs->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return vtts_reverb_stream_push(ctx, rs, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, st);
  });
}
