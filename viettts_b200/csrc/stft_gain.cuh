// The per-bin gain STFT of the bias denoiser (denoise.cu) and the watermark embedder (watermark.cu): n_fft 1024 / hop
// 256 / periodic Hann, centered frames with reflect padding 512 (F = n / 256 + 1 frames, frame f covers samples
// 256 f - 512 .. 256 f + 511), Y_f[k] = gain(k, f, X_f[k]) on bins 0..512, then the overlap-add of w * irfft(Y_f) over
// the envelope sum_f w^2 (vtts_denoise_ola).  Rows of <= 512 samples cannot be reflect-padded and are copied.
//
// Frame kernel.  One warp per frame, transformed alone (stftc): a frame's output bits are a function of its own 1024
// input samples, its absolute index and the gain, so the stream recomputes the frames an earlier push already used and
// gets the one-shot bits.  The gain is a policy: `float2 operator()(int k, long long f, float2 X) const` on the device.
//
// Stream.  Per slot a window of CARRY = 2048 carried inputs plus one chunk; an output t is emitted once the frames covering
// it are final, i.e. after 256 floor(t / 256) + 1024 inputs: before END a slot that has received P samples has emitted
// min(P, 256 max(0, floor(P / 256) - 3)).
#pragma once

#include <algorithm>
#include <vector>

#include "stft_common.cuh"
#include "stream_common.cuh"

namespace stftg {

constexpr int NF = vc::NFFT;      // 1024
constexpr int NB = vc::NBINS;     // 513
constexpr int HOP = vc::HOP;      // 256
constexpr int PAD = NF / 2;       // 512
constexpr int WARPS = 4;          // frames per CTA
constexpr int TP = stftc::TP;     // transpose pitch (float2)
constexpr int CARRY = 2048;       // carried inputs per stream slot (the frames of a push start at most 1791 before P0)
constexpr int LOOKAHEAD = 1023;

// rows == nullptr: the one-shot bounds of row b: n = n_in[b] clamped to [0, S] (or S), all S outputs written (zeros
// past n), frames 0 .. n / 256 when n > 512
__device__ __forceinline__ DnRow frame_row(const DnRow* rows, const int* n_in, int S, int b) {
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

template <class Gain>
__global__ void __launch_bounds__(WARPS * 32) gain_frame_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                 const int* __restrict__ n_in, const DnRow* __restrict__ rows,
                                                                 const float* __restrict__ hann, const float2* __restrict__ tw,
                                                                 const Gain gain, float* __restrict__ ws, int ws_frames) {
  __shared__ float2 smem[WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, fl = blockIdx.x * WARPS + warp;
  const DnRow r = frame_row(rows, n_in, S, b);
  if (fl >= r.nfr) return;                               // warps are independent: no block-level barrier below
  float2* sw = smem + (size_t)warp * 32 * TP;
  const float* xr = x + (size_t)b * x_ld;
  const long long g = r.g0 + fl;
  const long long j0 = g * HOP - PAD;

  // ---- windowed frame: sample j0 + lane + 32 m, reflected at 0 and n - 1 of the row ----
  float2 v[32];
  stftc::read_frame(v, xr, r.x0, r.n, j0, hann, lane);
  stftc::fft1024(v, sw, tw, lane);

  // ---- gain on bins k = lane + 32 k2 <= 512 ----
  __syncwarp();                                          // every lane has read sw
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k = lane + 32 * fftc::bitrev5(p);
    if (k <= NB - 1) sw[k] = gain(k, g, v[p]);
  }
  __syncwarp();

  // ---- inverse: w * irfft(Y) of the gained spectrum ----
  stftc::inverse_frame(v, sw, tw, lane);
  stftc::write_frame(v, hann, lane, ws + ((size_t)b * ws_frames + fl) * NF);
}

// frames then overlap-add: two launches
template <class Gain>
int launch(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const DnRow* rows, int B, long long max_frames,
           long long max_out, const Gain& gain, float* ws, int ws_frames, float* y, long long y_ld, cudaStream_t st) {
  const float2* tw = reinterpret_cast<const float2*>(ctx->fft_tw);
  const unsigned fgrid = (unsigned)std::max(1LL, (max_frames + WARPS - 1) / WARPS);
  gain_frame_kernel<Gain><<<dim3(fgrid, B), WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, ctx->hann, tw, gain, ws, ws_frames);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return vtts_denoise_ola(ctx, x, x_ld, S, n_in, rows, B, max_out, ws, ws_frames, y, y_ld, st);
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct Stream : SampleStream<DnRow> {
  int out_pitch = 0, ws_frames = 0;
  float* ws = nullptr;          // frame workspace [S][ws_frames][1024]

  Stream(vtts_ctx* c, int s, int f) : SampleStream(c, s, f, CARRY) {
    // outputs per push: fewer than n_new + 256 before END, at most n_new + 1023 with it (E(P0) >= P0 - 1023)
    out_pitch = f + LOOKAHEAD;
    // frames per push: outputs [E0, E1) read frames floor((E0 - 511) / 256) .. floor((E1 + 511) / 256)
    ws_frames = (out_pitch + 2 * PAD) / HOP + 2;
  }
  void carve_ws(Arena& a) { ws = a.take<float>((size_t)S * ws_frames * NF); }

  // After the arguments are checked: the push's rows and outputs [E0, E1) per slot (E1 into e1, counts into n_out),
  // uploaded with the window step, then the two launches of `gain`.  copy: every row's outputs are its inputs.
  template <class Gain>
  int push(const char* who, const float* x_dev, const int32_t* n_new, const uint8_t* flags, float* y_dev, int32_t* n_out,
           const Gain& gain, bool copy, cudaStream_t st) {
    DnRow* rw = rows<0>();
    std::vector<long long> E1(S);
    long long max_out = 0, max_frames = 0;
    for (int s = 0; s < S; ++s) {
      const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
      const long long P0 = begin ? 0 : slots.P[s], E0 = begin ? 0 : slots.E[s], P1 = P0 + n_new[s];
      long long e = E0;
      if (act) e = end ? P1 : std::min(P1, (long long)HOP * std::max(0LL, P1 / HOP - 3));
      E1[s] = e;
      n_out[s] = (int32_t)(e - E0);
      DnRow r{};
      r.x0 = P0 - CARRY;
      r.n = end ? P1 : DN_OPEN;
      r.e0 = E0;
      r.cnt = e - E0;
      r.copy = copy || (end && P1 <= PAD);
      if (r.cnt > 0 && !r.copy) {
        const long long p0 = E0 + PAD, p1 = e - 1 + PAD;
        r.g0 = p0 >= NF - 1 ? (p0 - (NF - 1) + HOP - 1) / HOP : 0;
        r.nfr = (int)(std::min(r.n / HOP, p1 / HOP) - r.g0 + 1);
      }
      if (r.nfr > ws_frames || r.cnt > out_pitch)
        return ctx->fail(VTTS_ERR_CUDA, "%s: slot %d needs %d frames / %lld outputs (internal bound %d / %d)", who, s, r.nfr, r.cnt,
                         ws_frames, out_pitch);
      rw[s] = r;
      max_out = std::max(max_out, r.cnt);
      max_frames = std::max(max_frames, (long long)r.nfr);
    }

    // ---- device: one table copy, prep, frames, overlap-add (three launches) ----
    int rc = upload(n_new, flags, x_dev, st);
    if (rc) return rc;
    rc = launch(ctx, win, cap, cap, nullptr, d_rows<0>(), S, max_frames, max_out, gain, ws, ws_frames, y_dev, out_pitch, st);
    if (rc) return rc;
    slots.commit(n_new, flags, E1.data());
    return VTTS_OK;
  }
};

}  // namespace stftg
