// Phase vocoder: a peak-locked phase vocoder (Laroche & Dolson 1999) on the denoiser's STFT, fp32 on the device in every
// vtts_precision mode, with the phase recurrence in double.  It serves two calls, the pitch shifter and the time
// stretcher, which differ in where the analysis frames sit, in one coefficient of the recurrence and in the bin remap.
//   STFT n_fft 1024 / periodic Hann / reflect padding 512; analysis frame t centred at a_t | X_t, a = |X_t|, theta =
//   arg X_t | peaks: a[k] > a[k-1], a[k] >= a[k+1], a[k] > 0 (neighbours outside [0, 512] count as -1) | every bin
//   belongs to its nearest peak, the lower one on a tie | h_t = a_t - a_t-1 |
//   omega_t[p] = 2 pi p / N + princarg(theta_t[p] - theta_t-1[p] - 2 pi p h_t / N) / h_t (2 pi p / N at t = 0) |
//   psi_t(p) = princarg(psi_t-1[p] + (H r - h_t) omega_t[p]) with h_0 = H = 256, psi_t-1[k] the rotation of the peak
//   that owned bin k in frame t - 1 (0 before frame 0 and in a frame without peaks) | bin k of peak p moves to
//   k + D_p, D_p = rint((r - 1) p), times (-1)^D_p e^(i psi_t(p)), targets outside [0, 512] dropped, contributions summed
//   in ascending k | the denoiser's inverse and overlap-add over the synthesis frames at hop H.
// Pitch shift: a_t = 256 t, F = n / 256 + 1 frames, r = fp32(2^(s / 12)), s in [-12, 12]; n outputs.  (H r - 256) equals
//   H (r - 1) exactly in double.  Rows with s == 0, and rows of <= 512 samples, are copied.
// Voice shift: the pitch shift with a formant shift phi (finite, in [-12, 12]) or none (the formants follow the pitch,
//   the pitch shift above bit for bit).  f = fp32(2^(phi / 12)).  Per analysis frame the cepstral envelope of a = |X_t|:
//   m = max a, l[k] = ln max(a[k], 1e-4 m, 1e-30), c[q] = (l[0] + (-1)^q l[512] + 2 sum_k=1..511 l[k] cos(2 pi k q / N)) / N
//   for q = 0..26, E[k] = c[0] + 2 sum_q=1..26 c[q] cos(2 pi k q / N) (cosines from the FFT twiddle table at k q mod N);
//   bin k landing on t = k + D_p is multiplied after its rotation by exp(min(E(t / f) - E[k], ln 10^(24 / 20))), E(u)
//   linear between E[floor u] and E[floor u + 1], E[512] past 512, u = t / f in double.  Rows with s == 0 and phi in
//   {none, 0}, and rows of <= 512 samples, are copied; s == 0 with phi != 0 runs the vocoder at r = 1.
// Time stretch: tempo alpha (fp32, in [0.5, 2], > 1 faster); M = floor(n / (double)alpha + 0.5) outputs, T = M / 256 + 1
//   frames, a_t = min(rint(256 t (double)alpha), n - 1), r = 1 (so D_p = 0 and psi_0 = 0).  h_t >= 1: a_t rises by at
//   least 128 until the clamp, and only the last frame can reach it (256 (T - 2) alpha <= n + 1 - 128).  Rows with
//   alpha == 1, and rows of <= 512 samples, give their first min(n, M) samples, then zeros up to M.
//
// Analysis kernel.  One warp per frame, as denoise_frame_kernel: the frame is read and transformed ALONE, so its
// outputs (X, theta in double, the owner map) are a function of its own 1024 input samples.
// Phase kernel.  One CTA per row, one thread per bin, walks the row's frames in order: the only sequential part.  A peak
// thread computes its rotation into shared memory; after one barrier every bin takes its owner's.  Double buffering of
// the shared rotations makes that one barrier per frame.
// Synthesis kernel.  One warp per frame: the rotated bins and their targets go to shared memory, lane l then sums the
// targets [16 l, 16 l + 16) over the sources in ascending order, and the denoiser's inverse transform windows the frame.
// Overlap-add.  denoise_ola_kernel itself (vtts_denoise_ola), over the synthesis frames into the outputs.
// Envelope.  The analysis and synthesis kernels take a compile-time flag; the legacy instantiations (no row has a formant
// shift) compile as before.  With it, the analysis warp of a row with f != 0 forms E after the owners: lane l takes the
// bins [16 l, 16 l + 16) (lane 31 also 512); m by a max-shuffle; each c[q] is the lane's fmaf sum over its bins in
// ascending order of weight * l[k] * cos (weight 1 at k = 0 and 512, else 2), then an xor-shuffle tree at distances 16,
// 8, 4, 2, 1, times 1 / 1024; each E[k] is c[0] + 2 s, s the fmaf sum over q = 1..26 ascending.  The synthesis warp
// multiplies each rotated bin by its gain (fp32 interpolation fmaf(frac, E[i + 1] - E[i], E[i]), expf) before the scatter.
//
// Streams.  Per slot the denoiser's window (2048 carried inputs plus one chunk), the 64-bit position, the next unscanned
// frame, theta and psi (double) of the last scanned frame, and the synthesized frames later outputs still overlap, in
// two halves that alternate per push (the carried frames are copied from the other half by the synthesis kernel).  A
// frame is scanned once it reads no input past the ones received (a_t + 512 <= P, and P > 512 for frame 0's
// reflection), or at END; such frames never reach the end clamp or the far reflection, so they equal the one-shot
// call's.  A frame scanned in a push starts past P0 - 1024 (it was not scannable at P0), so 2048 carried inputs cover
// every tempo, alpha = 2 included.  The pitch shifter releases outputs on the denoiser's schedule; the time stretcher
// releases output u once every synthesis frame that weighs it (256 g < u + 512 <= 256 g + 1023; the overlap-add skips
// the zero-weight sample 0 of a frame) is synthesized: max(0, 256 Q - 511) after Q scanned frames (frame Q - 1 exists
// in the final row, M >= 256 Q), everything at END, and alpha == 1 slots (copies) everything received.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "stft_common.cuh"
#include "stream_common.cuh"

namespace {

constexpr int NF = vc::NFFT;      // 1024
constexpr int NB = vc::NBINS;     // 513
constexpr int HOP = vc::HOP;      // 256
constexpr int PAD = NF / 2;       // 512
constexpr int TP = stftc::TP;
constexpr int PS_WARPS = 4;       // frames per CTA of the analysis and synthesis kernels
constexpr int PH_THREADS = 544;   // phase kernel: one thread per bin (17 warps)
constexpr int OWN_LD = 514;       // pitch of the int16 owner rows
constexpr int PS_K = 2048;        // carried inputs per stream slot (as the denoise stream)
constexpr int PS_LOOKAHEAD = 1023;
constexpr int TS_LOOKAHEAD = 1536;  // before END a time-stretch slot has released more than P / alpha - 1536 outputs
constexpr double TWO_PI = 6.283185307179586;
constexpr int ENV_Q = 26;                          // cepstral lifter: c[0..26]
constexpr float ENV_CAP = 2.7631021115928547f;     // ln 10^(24 / 20): the largest boost of a bin

struct PsShift {
  float r;            // pitch: fp32(2^(s / 12)); time stretch: 1
  float tempo;        // time stretch: alpha; pitch: 0 (frames at 256 t, no end clamp)
  int copy;           // s == 0 with the formants following the pitch or unmoved, or alpha == 1
};

struct PsRow {
  long long x0;       // absolute index of input buffer element 0
  long long n;        // row length (DN_OPEN while a stream slot is open)
  long long m;        // outputs of the row: n (pitch) or M (time stretch)
  long long q0;       // first frame this call scans (analysis, phase step, synthesis)
  long long fb;       // first frame of the synthesized-frame buffer this call fills
  long long fb_prev;  // stream: first frame of the slot's other half; frames [fb, q0) are copied from it
  int nq;             // frames scanned
  int nsyn;           // frames of the buffer: [fb, fb + nsyn)
  int half;           // stream: the half of the slot's frame buffer this call fills
  int copy;           // the outputs are the inputs
  float r;            // ratio
  float tempo;        // as PsShift::tempo
};

// workspace of one call: per row `fr` analysed frames and `halves` x `nbuf` synthesized frames
struct PsWs {
  float2* X;          // [rows][fr][513]
  double* th;         // [rows][fr][513]
  short* own;         // [rows][fr][OWN_LD]: the owning peak of each bin, -1 in a frame without peaks
  double* psi;        // [rows][fr][513]: the owner's rotation
  float* syn;         // [rows][halves][nbuf][1024]: windowed time frames
  int fr, nbuf, halves;
};

// the voice shift's per-call additions, read only by the envelope instantiations (a separate argument, so the legacy
// kernels keep their parameter layout)
struct PsEnv {
  const float* ratio; // [rows]: f = fp32(2^(phi / 12)), or 0 where the formants follow the pitch
  float* env;         // [rows][fr][513]: E of each analysed frame
};

// M = floor(n / (double)alpha + 0.5): the time stretcher's output length
__host__ __device__ __forceinline__ long long ts_len(long long n, float tempo) { return (long long)floor((double)n / (double)tempo + 0.5); }
// rint(256 g (double)alpha): the unclamped centre of analysis frame g of the time stretcher
__host__ __device__ __forceinline__ long long ts_centre(long long g, float tempo) { return (long long)rint(256.0 * (double)g * (double)tempo); }

// centre a_g of analysis frame g
__device__ __forceinline__ long long ps_centre(const PsRow& r, long long g) {
  return r.tempo == 0.f ? g * HOP : min(ts_centre(g, r.tempo), r.n - 1);
}

// rows == nullptr: the one-shot bounds of row b, n = n_in[b] clamped to [0, S] (or S), every frame scanned in this call
__device__ __forceinline__ PsRow ps_row(const PsRow* rows, const int* n_in, const PsShift* shifts, int S, int b) {
  if (rows) return rows[b];
  PsRow r;
  r.n = n_in ? (long long)min(max(n_in[b], 0), S) : (long long)S;
  r.x0 = 0;
  r.q0 = 0;
  r.fb = 0;
  r.fb_prev = 0;
  r.half = 0;
  r.r = shifts[b].r;
  r.tempo = shifts[b].tempo;
  r.m = r.tempo == 0.f ? r.n : ts_len(r.n, r.tempo);
  r.copy = r.n <= PAD || shifts[b].copy;
  r.nq = r.copy ? 0 : (int)(r.m / HOP + 1);
  r.nsyn = r.nq;
  return r;
}

__device__ __forceinline__ double princarg(double x) { return x - TWO_PI * rint(x / TWO_PI); }

// E[0..512] of one frame into env from its magnitudes mag[0..512] (shared, synced over the warp), in the order the
// header states
__device__ __forceinline__ void ps_envelope(const float* mag, const float2* __restrict__ tw, int lane, float* __restrict__ env) {
  const int k0 = 16 * lane, cnt = lane == 31 ? 17 : 16;
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < 17; ++i)
    if (i < cnt) m = fmaxf(m, mag[k0 + i]);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
  const float lo = fmaxf(1e-4f * m, 1e-30f);
  float l[17];
#pragma unroll
  for (int i = 0; i < 17; ++i) {
    const int k = k0 + i;
    const float v = i < cnt ? logf(fmaxf(mag[k], lo)) : 0.f;
    l[i] = k == 0 || k == NB - 1 ? v : 2.f * v;
  }
  float c[ENV_Q + 1];
#pragma unroll
  for (int q = 0; q <= ENV_Q; ++q) {
    float p = 0.f;
#pragma unroll
    for (int i = 0; i < 17; ++i)
      if (i < cnt) p = fmaf(l[i], __ldg(&tw[((k0 + i) * q) & (NF - 1)].x), p);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) p += __shfl_xor_sync(0xffffffffu, p, d);
    c[q] = p * (1.f / NF);
  }
#pragma unroll
  for (int i = 0; i < 17; ++i) {
    if (i < cnt) {
      const int k = k0 + i;
      float s = 0.f;
#pragma unroll
      for (int q = 1; q <= ENV_Q; ++q) s = fmaf(c[q], __ldg(&tw[(k * q) & (NF - 1)].x), s);
      env[k] = c[0] + 2.f * s;
    }
  }
}

// the gain of a bin k landing on t: exp(min(E(t / f) - E[k], ln 10^(24 / 20)))
__device__ __forceinline__ float ps_gain(const float* __restrict__ env, int k, int t, float ratio) {
  const double u = (double)t / (double)ratio;
  float eu;
  if (u >= (double)(NB - 1)) {
    eu = env[NB - 1];
  } else {
    const int i = (int)u;
    const float e0 = env[i];
    eu = fmaf((float)(u - i), env[i + 1] - e0, e0);
  }
  return expf(fminf(eu - env[k], ENV_CAP));
}

template <bool ENV>
__global__ void __launch_bounds__(PS_WARPS * 32) pitch_analysis_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                      const int* __restrict__ n_in, const PsShift* __restrict__ shifts,
                                                                      const PsRow* __restrict__ rows, const float* __restrict__ hann,
                                                                      const float2* __restrict__ tw, PsWs w, PsEnv e) {
  __shared__ float2 smem[PS_WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, fl = blockIdx.x * PS_WARPS + warp;
  const PsRow r = ps_row(rows, n_in, shifts, S, b);
  if (fl >= r.nq) return;                                // warps are independent: no block-level barrier below
  float2* sw = smem + (size_t)warp * 32 * TP;
  float2 v[32];
  stftc::read_frame(v, x + (size_t)b * x_ld, r.x0, r.n, ps_centre(r, r.q0 + fl) - PAD, hann, lane);
  stftc::fft1024(v, sw, tw, lane);

  // ---- X, theta = atan2 in double, |X| into shared memory ----
  __syncwarp();                                          // every lane has read sw
  const size_t f = (size_t)b * w.fr + fl;
  float* mag = reinterpret_cast<float*>(sw);
#pragma unroll
  for (int p = 0; p < 32; ++p) {
    const int k = lane + 32 * fftc::bitrev5(p);
    if (k < NB) {
      const float2 X = v[p];
      w.X[f * NB + k] = X;
      w.th[f * NB + k] = atan2((double)X.y, (double)X.x);
      mag[k] = sqrtf(X.x * X.x + X.y * X.y);
    }
  }
  __syncwarp();

  // ---- peaks and owners: lane l holds bins [16 l, 16 l + 16), lane 31 also bin 512 ----
  constexpr int NONE_R = 1 << 20;
  const int k0 = 16 * lane, cnt = lane == 31 ? 17 : 16;
  unsigned pk = 0;
#pragma unroll
  for (int i = 0; i < 17; ++i) {
    const int k = k0 + i;
    if (i < cnt) {
      const float a = mag[k];
      const float lft = k > 0 ? mag[k - 1] : -1.f, rgt = k < NB - 1 ? mag[k + 1] : -1.f;
      if (a > lft && a >= rgt && a > 0.f) pk |= 1u << i;
    }
  }
  // nearest peak at or left of each segment's start (exclusive prefix max of the segments' last peaks) and at or right
  // of its end (exclusive suffix min of their first peaks)
  int last = pk ? k0 + 31 - __clz(pk) : -1, first = pk ? k0 + __ffs(pk) - 1 : NONE_R;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, last, d), dn = __shfl_down_sync(0xffffffffu, first, d);
    if (lane >= d) last = max(last, u);
    if (lane + d < 32) first = min(first, dn);
  }
  int lrun = __shfl_up_sync(0xffffffffu, last, 1), rrun = __shfl_down_sync(0xffffffffu, first, 1);
  if (lane == 0) lrun = -1;
  if (lane == 31) rrun = NONE_R;
  int lk[17];
#pragma unroll
  for (int i = 0; i < 17; ++i) {
    if (pk >> i & 1) lrun = k0 + i;
    lk[i] = lrun;
  }
  short* own = w.own + f * OWN_LD;
#pragma unroll
  for (int i = 16; i >= 0; --i) {
    if (i < cnt) {
      const int k = k0 + i;
      if (pk >> i & 1) rrun = k;
      const int L = lk[i];
      int o;
      if (L < 0) o = rrun == NONE_R ? -1 : rrun;
      else o = (rrun == NONE_R || k - L <= rrun - k) ? L : rrun;
      own[k] = (short)o;
    }
  }
  if constexpr (ENV) {
    if (e.ratio[b] != 0.f) ps_envelope(mag, tw, lane, e.env + f * NB);
  }
}

// state: stream [rows][2][513] (theta, psi of the last scanned frame) or nullptr; ola: one-shot, receives the rows'
// overlap-add bounds (y_cnt outputs per row); dec: [rows][dec_fr][513] decisions, 1 | (e < 0) << 1 at a peak whose
// wrapped phase deviation is e, 0 elsewhere (test hook)
__global__ void __launch_bounds__(PH_THREADS) pitch_phase_kernel(const int* __restrict__ n_in, const PsShift* __restrict__ shifts,
                                                                const PsRow* __restrict__ rows, int S, PsWs w, double* __restrict__ state,
                                                                DnRow* __restrict__ ola, long long y_cnt, int* __restrict__ dec, int dec_fr) {
  __shared__ double ps_sh[2][NB];
  const int b = blockIdx.x, k = threadIdx.x;
  const PsRow r = ps_row(rows, n_in, shifts, S, b);
  if (ola && k == 0) {
    DnRow d;
    d.x0 = 0;
    d.n = r.copy ? min(r.n, r.m) : r.m;
    d.g0 = 0;
    d.e0 = 0;
    d.cnt = y_cnt;
    d.nfr = r.nq;
    d.copy = r.copy;
    ola[b] = d;
  }
  if (r.nq == 0) return;                                 // uniform over the CTA
  const bool bin = k < NB;
  const double hr = HOP * (double)r.r;                   // the rotation advances by (H r - h_t) omega
  double thp = 0.0, psp = 0.0;
  if (state && bin) {
    thp = state[(size_t)b * 2 * NB + k];
    psp = state[(size_t)b * 2 * NB + NB + k];
  }
  const size_t f0 = (size_t)b * w.fr;
  int own = bin ? w.own[f0 * OWN_LD + k] : -1;
  double th = bin ? w.th[f0 * NB + k] : 0.0;
  long long a_prev = ps_centre(r, r.q0 - 1);
  for (int i = 0; i < r.nq; ++i) {
    const long long g = r.q0 + i;
    const long long a = ps_centre(r, g);
    int own_n = -1;
    double th_n = 0.0;
    if (bin && i + 1 < r.nq) {                           // the next frame's loads fly under this frame's step
      own_n = w.own[(f0 + i + 1) * OWN_LD + k];
      th_n = w.th[(f0 + i + 1) * NB + k];
    }
    int neg = 0;
    if (own == k) {
      const double h = g > 0 ? (double)(a - a_prev) : (double)HOP;
      double om = TWO_PI * k / NF, prev = 0.0;
      if (g > 0) {
        const double e = princarg(th - thp - TWO_PI * k * h / NF);
        neg = e < 0.0;
        om += e / h;
        prev = psp;
      }
      ps_sh[i & 1][k] = princarg(prev + (hr - h) * om);
    }
    __syncthreads();
    const double ps = own >= 0 ? ps_sh[i & 1][own] : 0.0;
    if (bin) {
      w.psi[(f0 + i) * NB + k] = ps;
      if (dec) dec[((size_t)b * dec_fr + g) * NB + k] = own == k ? 1 | neg << 1 : 0;
    }
    psp = ps;
    thp = th;
    own = own_n;
    th = th_n;
    a_prev = a;
  }
  if (state && bin) {
    state[(size_t)b * 2 * NB + k] = thp;
    state[(size_t)b * 2 * NB + NB + k] = psp;
  }
}

template <bool ENV>
__global__ void __launch_bounds__(PS_WARPS * 32) pitch_synth_kernel(const int* __restrict__ n_in, const PsShift* __restrict__ shifts,
                                                                   const PsRow* __restrict__ rows, int S, const float* __restrict__ hann,
                                                                   const float2* __restrict__ tw, PsWs w, PsEnv e) {
  __shared__ float2 smem[PS_WARPS * 32 * TP];            // per warp: Z[0..512], then the rotated bins [513..1025]
  __shared__ short tg_sh[PS_WARPS][NB + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, fl = blockIdx.x * PS_WARPS + warp;
  const PsRow r = ps_row(rows, n_in, shifts, S, b);
  if (fl >= r.nsyn) return;                              // warps are independent: no block-level barrier below
  const long long g = r.fb + fl;
  float* out = w.syn + (((size_t)b * w.halves + r.half) * w.nbuf + fl) * NF;
  if (g < r.q0) {                                        // synthesized by an earlier push: carried over from the other half
    const float4* src = reinterpret_cast<const float4*>(w.syn + (((size_t)b * w.halves + (1 - r.half)) * w.nbuf + (g - r.fb_prev)) * NF);
#pragma unroll
    for (int m = 0; m < NF / 128; ++m) reinterpret_cast<float4*>(out)[lane + 32 * m] = src[lane + 32 * m];
    return;
  }
  const size_t f = (size_t)b * w.fr + (g - r.q0);
  float2* sw = smem + (size_t)warp * 32 * TP;
  float2* rot = sw + NB;
  short* tg = tg_sh[warp];
  const double r1 = (double)r.r - 1.0;
  float fr = 0.f;
  const float* env = nullptr;
  if constexpr (ENV) {
    fr = e.ratio[b];
    env = e.env + f * NB;
  }
  for (int k = lane; k < NB; k += 32) {
    const int p = w.own[f * OWN_LD + k];
    int t = -1;
    float2 z = make_float2(0.f, 0.f);
    if (p >= 0) {
      const int d = (int)rint(r1 * p);
      if (k + d >= 0 && k + d < NB) {
        t = k + d;
        double sn, cs;
        sincos(w.psi[f * NB + k], &sn, &cs);
        z = fftc::cmul(w.X[f * NB + k], make_float2((float)cs, (float)sn));
        if (d & 1) z = make_float2(-z.x, -z.y);          // (-1)^D: the phase referred to the frame centre
        if constexpr (ENV) {
          if (fr != 0.f) {
            const float g = ps_gain(env, k, t, fr);
            z = make_float2(z.x * g, z.y * g);
          }
        }
      }
    }
    rot[k] = z;
    tg[k] = (short)t;
    sw[k] = make_float2(0.f, 0.f);
  }
  __syncwarp();
  const int lo = 16 * lane, hi = lane == 31 ? NB : lo + 16;
  for (int k = 0; k < NB; ++k) {
    const int t = tg[k];
    if (t >= lo && t < hi) {
      const float2 a = sw[t], c = rot[k];
      sw[t] = make_float2(a.x + c.x, a.y + c.y);
    }
  }
  __syncwarp();
  float2 v[32];
  stftc::inverse_frame(v, sw, tw, lane);
  stftc::write_frame(v, hann, lane, out);
}

bool shift_ok(float s) { return std::isfinite(s) && s >= -12.f && s <= 12.f; }
bool tempo_ok(float a) { return std::isfinite(a) && a >= 0.5f && a <= 2.f; }

int ps_check_shifts(vtts_ctx* ctx, const char* who, const float* semitones, int n) {
  if (!semitones) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null semitones", who);
  for (int i = 0; i < n; ++i)
    if (!shift_ok(semitones[i]))
      return ctx->fail(VTTS_ERR_BAD_ARG, "%s: semitones[%d] = %g (finite, in [-12, 12])", who, i, (double)semitones[i]);
  return VTTS_OK;
}

// formants: null (every row follows the pitch) or n formant shifts, finite and in [-12, 12]
int ps_check_formants(vtts_ctx* ctx, const char* who, const float* formants, int n) {
  if (formants)
    for (int i = 0; i < n; ++i)
      if (!shift_ok(formants[i]))
        return ctx->fail(VTTS_ERR_BAD_ARG, "%s: formants[%d] = %g (finite, in [-12, 12])", who, i, (double)formants[i]);
  return VTTS_OK;
}

int ts_check_tempos(vtts_ctx* ctx, const char* who, const float* tempo, int n) {
  if (!tempo) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null tempo", who);
  for (int i = 0; i < n; ++i)
    if (!tempo_ok(tempo[i])) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: tempo[%d] = %g (finite, in [0.5, 2])", who, i, (double)tempo[i]);
  return VTTS_OK;
}

// fp32(2^(s / 12)), computed in double and rounded once
float ps_ratio(float s) { return (float)std::pow(2.0, (double)s / 12.0); }
// phi: the formant shift, NaN where the formants follow the pitch; s == 0 copies unless the formants move
PsShift ps_params(float s, float phi = NAN) { return PsShift{ps_ratio(s), 0.f, s == 0.f && (std::isnan(phi) || phi == 0.f)}; }
PsShift ts_params(float tempo) { return PsShift{1.f, tempo, tempo == 1.f}; }
// the envelope ratio f of a row: 0 (no envelope) where the formants follow the pitch or the row is a copy
float ps_env_ratio(float phi, const PsShift& h) { return std::isnan(phi) || h.copy ? 0.f : ps_ratio(phi); }

void ps_carve(Arena& a, PsWs& w, int rows) {
  w.X = a.take<float2>((size_t)rows * w.fr * NB);
  w.th = a.take<double>((size_t)rows * w.fr * NB);
  w.own = a.take<short>((size_t)rows * w.fr * OWN_LD);
  w.psi = a.take<double>((size_t)rows * w.fr * NB);
  w.syn = a.take<float>((size_t)rows * w.halves * w.nbuf * NF);
}
float* ps_carve_env(Arena& a, const PsWs& w, int rows) { return a.take<float>((size_t)rows * w.fr * NB); }

// analysis, phase, synthesis (three launches); the synthesis is skipped when only the decisions are wanted.  env: the
// envelope instantiations with these buffers, or null for the legacy ones
int ps_launch(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const PsShift* shifts, const PsRow* rows, int B,
              long long max_nq, long long max_nsyn, const PsWs& w, double* state, DnRow* ola, long long y_cnt, int* dec, int dec_fr,
              const PsEnv* env, cudaStream_t st) {
  const float2* tw = reinterpret_cast<const float2*>(ctx->fft_tw);
  const PsEnv e = env ? *env : PsEnv{};
  const unsigned agrid = (unsigned)std::max(1LL, (max_nq + PS_WARPS - 1) / PS_WARPS);
  if (env) pitch_analysis_kernel<true><<<dim3(agrid, B), PS_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, shifts, rows, ctx->hann, tw, w, e);
  else pitch_analysis_kernel<false><<<dim3(agrid, B), PS_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, shifts, rows, ctx->hann, tw, w, e);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  pitch_phase_kernel<<<B, PH_THREADS, 0, st>>>(n_in, shifts, rows, S, w, state, ola, y_cnt, dec, dec_fr);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  if (dec) return VTTS_OK;
  const unsigned sgrid = (unsigned)std::max(1LL, (max_nsyn + PS_WARPS - 1) / PS_WARPS);
  if (env) pitch_synth_kernel<true><<<dim3(sgrid, B), PS_WARPS * 32, 0, st>>>(n_in, shifts, rows, S, ctx->hann, tw, w, e);
  else pitch_synth_kernel<false><<<dim3(sgrid, B), PS_WARPS * 32, 0, st>>>(n_in, shifts, rows, S, ctx->hann, tw, w, e);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// the pointer rejections of a one-shot call into y_dev, or dec_dev for the decisions test hook
int ps_pointers(vtts_ctx* ctx, const char* who, const float* x_dev, const float* y_dev, const int* dec_dev) {
  if (!x_dev || (!y_dev && !dec_dev)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: y must not alias x", who);
  return VTTS_OK;
}

// one-shot call (dec == nullptr) or the decisions test hook, on checked arguments: rows with the parameters h, F
// analysis frames for the longest row, Sy outputs per row; ratio: each row's envelope ratio (ps_env_ratio), or empty
// for the legacy kernels
int ps_one_shot(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const std::vector<PsShift>& h, long long F, int Sy,
                float* y_dev, int* dec_dev, cudaStream_t st, const std::vector<float>& ratio = {}) {
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const bool use_env = !ratio.empty();
  PsWs w{};
  w.fr = (int)F;
  w.nbuf = (int)F;
  w.halves = 1;
  Arena m(nullptr, 0, true);
  m.take<PsShift>(B);
  m.take<DnRow>(B);
  ps_carve(m, w, B);
  if (use_env) {
    m.take<float>(B);
    ps_carve_env(m, w, B);
  }
  rc = ctx->ensure_ws(m.off);
  if (rc) return rc;
  Arena a(ctx->ws, ctx->ws_bytes, false);
  PsShift* shifts = a.take<PsShift>(B);
  DnRow* ola = a.take<DnRow>(B);
  ps_carve(a, w, B);
  PsEnv env{};
  if (use_env) {
    float* r = a.take<float>(B);
    env.ratio = r;
    env.env = ps_carve_env(a, w, B);
    VTTS_CUDA(cudaMemcpyAsync(r, ratio.data(), (size_t)B * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  // pageable source: the call returns once the table is staged
  VTTS_CUDA(cudaMemcpyAsync(shifts, h.data(), (size_t)B * sizeof(PsShift), cudaMemcpyHostToDevice, st));
  if (dec_dev) {
    VTTS_CUDA(cudaMemsetAsync(dec_dev, 0, (size_t)B * F * NB * sizeof(int), st));
    return ps_launch(ctx, x_dev, S, S, n_dev, shifts, nullptr, B, F, F, w, nullptr, nullptr, 0, dec_dev, (int)F, nullptr, st);
  }
  rc = ps_launch(ctx, x_dev, S, S, n_dev, shifts, nullptr, B, F, F, w, nullptr, ola, Sy, nullptr, 0, use_env ? &env : nullptr, st);
  if (rc) return rc;
  return vtts_denoise_ola(ctx, x_dev, S, S, nullptr, ola, B, Sy, w.syn, w.nbuf, y_dev, Sy, st);
}

// the batch shape and per-row parameters h of a one-shot call of entry point `who`; formants: null (the pitch shift:
// legacy kernels) or one formant shift per row (the envelope kernels, each row's envelope ratio in `ratio`)
int ps_args(vtts_ctx* ctx, const char* who, int B, int S, const float* semitones, const float* formants, std::vector<PsShift>* h,
            std::vector<float>* ratio) {
  int rc = batch_check(ctx, who, B, S, S_ANY);
  if (!rc) rc = ps_check_shifts(ctx, who, semitones, B);
  if (!rc) rc = ps_check_formants(ctx, who, formants, B);
  if (rc) return rc;
  h->resize(B);
  ratio->resize(formants ? B : 0);
  for (int b = 0; b < B; ++b) {
    const float phi = formants ? formants[b] : NAN;
    (*h)[b] = ps_params(semitones[b], phi);
    if (formants) (*ratio)[b] = ps_env_ratio(phi, (*h)[b]);
  }
  return VTTS_OK;
}

int ps_call(vtts_ctx* ctx, const char* who, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones,
            const float* formants, float* y_dev, int* dec_dev, cudaStream_t st) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  std::vector<PsShift> h;
  std::vector<float> ratio;
  int rc = ps_args(ctx, who, B, S, semitones, formants, &h, &ratio);
  if (!rc) rc = ps_pointers(ctx, who, x_dev, y_dev, dec_dev);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, st);
  return ps_one_shot(ctx, x_dev, n_dev, B, S, h, S / HOP + 1, S, y_dev, dec_dev, st, ratio);
}

int ps_call_host(vtts_ctx* ctx, const char* who, const float* x, const int32_t* n_in, int B, int S, const float* semitones,
                 const float* formants, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  std::vector<PsShift> h;
  std::vector<float> ratio;
  int rc = ps_args(ctx, who, B, S, semitones, formants, &h, &ratio);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows(who, x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return ps_one_shot(ctx, hs.x(), hs.n(), B, S, h, S / HOP + 1, S, hs.dev<float>(o_y), nullptr, st, ratio); });
}

// frames of the longest time-stretched row of S samples: max over the rows of M(S) / 256 + 1
long long ts_frames(const float* tempo, int B, int S) {
  long long F = 1;
  for (int b = 0; b < B; ++b) F = std::max(F, ts_len(S, tempo[b]) / HOP + 1);
  return F;
}

// the batch shape, output row length Sy and per-row parameters h of a one-shot call of entry point `who`
int ts_args(vtts_ctx* ctx, const char* who, int B, int S, const float* tempo, int Sy, std::vector<PsShift>* h) {
  int rc = batch_check(ctx, who, B, S, S_ANY);
  if (!rc && Sy < 1) rc = ctx->fail(VTTS_ERR_BAD_ARG, "%s: Sy=%d (>= 1)", who, Sy);
  if (!rc) rc = ts_check_tempos(ctx, who, tempo, B);
  if (rc) return rc;
  h->resize(B);
  for (int b = 0; b < B; ++b) (*h)[b] = ts_params(tempo[b]);
  return VTTS_OK;
}

int ts_call(vtts_ctx* ctx, const char* who, const float* x_dev, const int32_t* n_dev, int B, int S, const float* tempo, float* y_dev, int Sy,
            int* dec_dev, cudaStream_t st) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  std::vector<PsShift> h;
  int rc = ts_args(ctx, who, B, S, tempo, y_dev ? Sy : 1, &h);   // the decisions hook has no output rows
  if (!rc) rc = ps_pointers(ctx, who, x_dev, y_dev, dec_dev);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, st);
  return ps_one_shot(ctx, x_dev, n_dev, B, S, h, ts_frames(tempo, B, S), Sy, y_dev, dec_dev, st);
}

}  // namespace

int vtts_pitch_shift_stream_lookahead(void) { return PS_LOOKAHEAD; }

int vtts_pitch_shift(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, float* y_dev,
                     void* stream) {
  if (ctx && !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift: null pointer");
  return ps_call(ctx, "pitch_shift", x_dev, n_dev, B, S, semitones, nullptr, y_dev, nullptr, (cudaStream_t)stream);
}

int vtts_voice_shift(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, const float* formants,
                     float* y_dev, void* stream) {
  if (ctx && !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "voice_shift: null pointer");
  return ps_call(ctx, "voice_shift", x_dev, n_dev, B, S, semitones, formants, y_dev, nullptr, (cudaStream_t)stream);
}

int vtts_debug_pitch_decisions(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, int32_t* dec_dev,
                               void* stream) {
  if (ctx && !dec_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_pitch_decisions: null pointer");
  return ps_call(ctx, "debug_pitch_decisions", x_dev, n_dev, B, S, semitones, nullptr, nullptr, dec_dev, (cudaStream_t)stream);
}

int vtts_pitch_shift_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* semitones, float* y) {
  return ps_call_host(ctx, "pitch_shift_host", x, n_in, B, S, semitones, nullptr, y);
}

int vtts_voice_shift_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* semitones, const float* formants,
                          float* y) {
  return ps_call_host(ctx, "voice_shift_host", x, n_in, B, S, semitones, formants, y);
}

int64_t vtts_time_stretch_length(int64_t n, float tempo) { return n < 0 || !tempo_ok(tempo) ? -1 : ts_len(n, tempo); }

int vtts_time_stretch_stream_lookahead(void) { return TS_LOOKAHEAD; }

int vtts_time_stretch(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* tempo, float* y_dev, int Sy,
                      void* stream) {
  if (ctx && !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "time_stretch: null pointer");
  return ts_call(ctx, "time_stretch", x_dev, n_dev, B, S, tempo, y_dev, Sy, nullptr, (cudaStream_t)stream);
}

int vtts_debug_time_stretch_decisions(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* tempo,
                                      int32_t* dec_dev, void* stream) {
  if (ctx && !dec_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_time_stretch_decisions: null pointer");
  return ts_call(ctx, "debug_time_stretch_decisions", x_dev, n_dev, B, S, tempo, nullptr, 0, dec_dev, (cudaStream_t)stream);
}

int vtts_time_stretch_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* tempo, float* y, int Sy) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  std::vector<PsShift> h;
  int rc = ts_args(ctx, "time_stretch_host", B, S, tempo, Sy, &h);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("time_stretch_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * Sy * 4, y);
  return hs.run([&](cudaStream_t st) {
    return ps_one_shot(ctx, hs.x(), hs.n(), B, S, h, ts_frames(tempo, B, S), Sy, hs.dev<float>(o_y), nullptr, st);
  });
}

// ---- streams ---------------------------------------------------------------------------------------------------
// One implementation serves both vocoder streams; `stretch` selects the time stretcher's frame positions and schedule.
// Push tables: the overlap-add rows, the vocoder rows and each slot's envelope ratio (PsEnv::ratio).
struct PvStream : SampleStream<DnRow, PsRow, float> {
  using SampleStream::SampleStream;
  int out_pitch = 0;
  bool stretch = false;
  PsWs w{};
  double* state = nullptr;      // [S][2][513]
  float* env = nullptr;         // pitch: [S][fr][513] (PsEnv::env)
  // per slot besides the shared state: next unscanned frame, first frame and half of the last push's synthesized-frame
  // buffer, shift or tempo since BEGIN, formant shift since BEGIN (NaN: the formants follow the pitch)
  std::vector<long long> q, fb;
  std::vector<int> half;
  std::vector<float> par, fpar;
};
struct vtts_pitch_shift_stream : PvStream {
  using PvStream::PvStream;
};
struct vtts_time_stretch_stream : PvStream {
  using PvStream::PvStream;
};

namespace {

// frames scanned per push (at most fr), outputs per push (out_pitch) and the slots' neutral parameter
template <class Stream>
int pv_create(vtts_ctx* ctx, const char* who, int max_streams, int max_chunk_samples, bool stretch, Stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, who, out, out_pitch != nullptr, max_streams, max_chunk_samples);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const int S = max_streams;
  std::unique_ptr<Stream> ps(new Stream(ctx, S, max_chunk_samples, PS_K));
  ps->stretch = stretch;
  if (!stretch) {
    ps->out_pitch = max_chunk_samples + PS_LOOKAHEAD;  // as the denoise stream
    // frames scanned per push: at most n_new / 256 + 3 (with END); the buffer also holds the <= 3 carried frames
    ps->w.fr = max_chunk_samples / HOP + 4;
  } else {
    // outputs per push: at most 2 n_new + 256 before END, (n_new + 512.5) / alpha + 512.5 with it; frames scanned: at
    // most n_new / 128 + 1 before END, (n_new + 512.5) / (256 alpha) + 2.01 with it
    ps->out_pitch = 2 * max_chunk_samples + 2048;
    ps->w.fr = max_chunk_samples / 128 + 8;
  }
  ps->w.nbuf = ps->w.fr + 4;
  ps->w.halves = 2;
  ps->q.assign(S, 0);
  ps->fb.assign(S, 0);
  ps->half.assign(S, 0);
  ps->par.assign(S, stretch ? 1.f : 0.f);
  ps->fpar.assign(S, NAN);
  rc = stream_alloc(ctx, who, *ps, [&](Arena& a) {
    ps->carve_window(a);
    ps_carve(a, ps->w, S);
    if (!stretch) ps->env = ps_carve_env(a, ps->w, S);
    ps->state = a.take<double>((size_t)S * 2 * NB);
    ps->carve_tables(a);
  });
  if (rc) return rc;
  *out_pitch = ps->out_pitch;
  *out = ps.release();
  return VTTS_OK;
}

// par: semitones (pitch) or tempo (time stretch) per slot, read with BEGIN; fmt (pitch only): formant shifts per slot,
// read with BEGIN (null: the slots that begin follow the pitch), for an open slot its formant shift or NaN where it
// follows the pitch
int pv_push(vtts_ctx* ctx, const char* who, PvStream* ps, const float* x_dev, const int32_t* n_new, const uint8_t* flags, const float* par,
            const float* fmt, float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, who, ps, x_dev && n_new && flags && y_dev && n_out);
  if (rc) return rc;
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: y must not alias x", who);
  const bool stretch = ps->stretch;
  rc = ps->slots.check(ctx, who, ps->F, n_new, flags, [&](int s) -> int {
    if (stretch) {
      if (flags[s] & 1) {
        if (!par) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: BEGIN needs the tempo array", who);
        if (!tempo_ok(par[s])) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: tempo[%d] = %g (finite, in [0.5, 2])", who, s, (double)par[s]);
      } else if (par && !(par[s] == ps->par[s])) {
        return ctx->fail(VTTS_ERR_BAD_ARG, "%s: tempo[%d] = %g, but slot %d runs at tempo %g until END (BEGIN to change it)", who, s,
                         (double)par[s], s, (double)ps->par[s]);
      }
      return VTTS_OK;
    }
    if (flags[s] & 1) {
      if (!par) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: BEGIN needs the semitones array", who);
      if (!shift_ok(par[s])) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: semitones[%d] = %g (finite, in [-12, 12])", who, s, (double)par[s]);
      if (fmt && !shift_ok(fmt[s])) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: formants[%d] = %g (finite, in [-12, 12])", who, s, (double)fmt[s]);
    } else if (par && !(par[s] == ps->par[s])) {
      return ctx->fail(VTTS_ERR_BAD_ARG, "%s: semitones[%d] = %g, but slot %d shifts by %g until END (BEGIN to change it)", who, s,
                       (double)par[s], s, (double)ps->par[s]);
    } else if (fmt && !(fmt[s] == ps->fpar[s] || (std::isnan(fmt[s]) && std::isnan(ps->fpar[s])))) {
      return ctx->fail(VTTS_ERR_BAD_ARG, "%s: formants[%d] = %g, but slot %d has formant shift %g until END (NaN: it follows the pitch; "
                       "BEGIN to change it)", who, s, (double)fmt[s], s, (double)ps->fpar[s]);
    }
    return VTTS_OK;
  });
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = ps->S;
  const SlotState& sl = ps->slots;

  // ---- host bookkeeping: outputs [E0, E1), frames [q0, q1) scanned, synthesized-frame buffer [fb, q1) ----
  DnRow* rows = ps->rows<0>();
  PsRow* prow = ps->rows<1>();
  float* eratio = ps->rows<2>();
  std::vector<long long> E1(S), Q1(S);
  long long max_out = 0, max_nq = 0, max_nsyn = 0;
  bool use_env = false;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : sl.P[s], E0 = begin ? 0 : sl.E[s], P1 = P0 + n_new[s];
    const float pv = begin ? par[s] : ps->par[s];
    const float fv = begin ? (fmt ? fmt[s] : NAN) : ps->fpar[s];
    const PsShift h = stretch ? ts_params(pv) : ps_params(pv, fv);
    eratio[s] = act && !stretch ? ps_env_ratio(fv, h) : 0.f;
    const long long M1 = end ? (stretch ? ts_len(P1, pv) : P1) : DN_OPEN;   // the row's outputs, once known
    DnRow r{};
    PsRow p{};
    r.x0 = p.x0 = P0 - PS_K;
    p.n = end ? P1 : DN_OPEN;
    p.m = M1;
    r.copy = p.copy = h.copy || (end && P1 <= PAD);
    r.n = end && r.copy ? std::min(P1, M1) : M1;
    p.r = h.r;
    p.tempo = h.tempo;
    const long long q0 = begin ? 0 : ps->q[s];
    long long q1 = q0;
    if (act && !p.copy) {
      if (end) {
        q1 = M1 / HOP + 1;
      } else if (!stretch) {
        q1 = P1 > PAD ? (P1 - PAD) / HOP + 1 : 0;
      } else {
        while (P1 > PAD && ts_centre(q1, pv) + PAD <= P1) ++q1;
      }
    }
    long long e = E0;
    if (act) {
      if (end) e = M1;
      else if (!stretch) e = std::min(P1, (long long)HOP * std::max(0LL, P1 / HOP - 3));
      else e = h.copy ? P1 : std::max(0LL, HOP * q1 - (PAD - 1));
    }
    E1[s] = e;
    n_out[s] = (int32_t)(e - E0);
    r.e0 = E0;
    r.cnt = e - E0;
    Q1[s] = q0;
    if (act && !p.copy) {
      const long long p0 = E0 + PAD;
      const long long fb = p0 >= NF - 1 ? (p0 - (NF - 1) + HOP - 1) / HOP : 0;
      p.q0 = q0;
      p.nq = (int)(q1 - q0);
      p.fb = fb;
      p.fb_prev = ps->fb[s];
      p.nsyn = (int)(q1 - fb);
      p.half = begin ? 0 : 1 - ps->half[s];
      r.g0 = fb - (long long)p.half * ps->w.nbuf;
      if (r.cnt > 0) r.nfr = (int)(std::min(r.n / HOP, (e - 1 + PAD) / HOP) - fb + 1);
      Q1[s] = q1;
      if (fb > q0 || q1 < q0 || (!begin && fb < ps->fb[s]) || p.nq > ps->w.fr || p.nsyn > ps->w.nbuf)
        return ctx->fail(VTTS_ERR_CUDA, "%s: slot %d frames [%lld, %lld) buffer from %lld (internal bound %d / %d)", who, s, q0, q1, fb,
                         ps->w.fr, ps->w.nbuf);
    }
    if (r.cnt > ps->out_pitch)
      return ctx->fail(VTTS_ERR_CUDA, "%s: slot %d needs %lld outputs (internal bound %d)", who, s, r.cnt, ps->out_pitch);
    rows[s] = r;
    prow[s] = p;
    max_out = std::max(max_out, r.cnt);
    max_nq = std::max(max_nq, (long long)p.nq);
    max_nsyn = std::max(max_nsyn, (long long)p.nsyn);
    use_env |= eratio[s] != 0.f && p.nq > 0;
  }

  // ---- device: table copy, window step, analysis, phase, synthesis, overlap-add (five launches) ----
  rc = ps->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  // the envelope kernels only when a slot scans a frame with its formants moved: the other slots' bits are the same in both
  const PsEnv env{ps->d_rows<2>(), ps->env};
  rc = ps_launch(ctx, ps->win, ps->cap, ps->cap, nullptr, nullptr, ps->d_rows<1>(), S, max_nq, max_nsyn, ps->w, ps->state, nullptr, 0, nullptr, 0,
                 use_env ? &env : nullptr, st);
  if (rc) return rc;
  rc = vtts_denoise_ola(ctx, ps->win, ps->cap, ps->cap, nullptr, ps->d_rows<0>(), S, max_out, ps->w.syn, 2 * ps->w.nbuf, y_dev, ps->out_pitch, st);
  if (rc) return rc;

  // ---- commit the slot state ----
  for (int s = 0; s < S; ++s) {
    if (!SlotState::active(n_new, flags, s)) continue;
    const bool begin = flags[s] & 1;
    if (begin) {
      ps->par[s] = par[s];
      ps->fpar[s] = fmt ? fmt[s] : NAN;
    }
    if (prow[s].nsyn > 0 || prow[s].nq > 0) {
      ps->fb[s] = prow[s].fb;
      ps->half[s] = prow[s].half;
    } else if (begin) {
      ps->fb[s] = 0;
      ps->half[s] = 0;
    }
    ps->q[s] = Q1[s];
  }
  ps->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

}  // namespace

int vtts_pitch_shift_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, vtts_pitch_shift_stream** out, int* out_pitch) {
  return pv_create(ctx, "pitch_shift_stream_create", max_streams, max_chunk_samples, false, out, out_pitch);
}

int vtts_pitch_shift_stream_destroy(vtts_ctx* ctx, vtts_pitch_shift_stream* ps) {
  return stream_destroy(ctx, "pitch_shift_stream_destroy", ps);
}

int vtts_pitch_shift_stream_push(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                 const float* semitones, float* y_dev, int32_t* n_out, void* stream) {
  return pv_push(ctx, "pitch_shift_stream_push", ps, x_dev, n_new, flags, semitones, nullptr, y_dev, n_out, stream);
}

int vtts_pitch_shift_stream_push_host(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x, const int32_t* n_new, const uint8_t* flags,
                                      const float* semitones, float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "pitch_shift_stream_push_host", ps, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ps->S * ps->F * 4), o_y = hs.out((size_t)ps->S * ps->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return pv_push(ctx, "pitch_shift_stream_push", ps, hs.dev<const float>(o_x), n_new, flags, semitones, nullptr, hs.dev<float>(o_y), n_out, st);
  });
}

int vtts_voice_shift_stream_push(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                 const float* semitones, const float* formants, float* y_dev, int32_t* n_out, void* stream) {
  return pv_push(ctx, "voice_shift_stream_push", ps, x_dev, n_new, flags, semitones, formants, y_dev, n_out, stream);
}

int vtts_voice_shift_stream_push_host(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x, const int32_t* n_new, const uint8_t* flags,
                                      const float* semitones, const float* formants, float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "voice_shift_stream_push_host", ps, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ps->S * ps->F * 4), o_y = hs.out((size_t)ps->S * ps->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return pv_push(ctx, "voice_shift_stream_push", ps, hs.dev<const float>(o_x), n_new, flags, semitones, formants, hs.dev<float>(o_y), n_out, st);
  });
}

int vtts_time_stretch_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, vtts_time_stretch_stream** out, int* out_pitch) {
  return pv_create(ctx, "time_stretch_stream_create", max_streams, max_chunk_samples, true, out, out_pitch);
}

int vtts_time_stretch_stream_destroy(vtts_ctx* ctx, vtts_time_stretch_stream* ts) {
  return stream_destroy(ctx, "time_stretch_stream_destroy", ts);
}

int vtts_time_stretch_stream_push(vtts_ctx* ctx, vtts_time_stretch_stream* ts, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                  const float* tempo, float* y_dev, int32_t* n_out, void* stream) {
  return pv_push(ctx, "time_stretch_stream_push", ts, x_dev, n_new, flags, tempo, nullptr, y_dev, n_out, stream);
}

int vtts_time_stretch_stream_push_host(vtts_ctx* ctx, vtts_time_stretch_stream* ts, const float* x, const int32_t* n_new,
                                       const uint8_t* flags, const float* tempo, float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "time_stretch_stream_push_host", ts, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ts->S * ts->F * 4), o_y = hs.out((size_t)ts->S * ts->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return pv_push(ctx, "time_stretch_stream_push", ts, hs.dev<const float>(o_x), n_new, flags, tempo, nullptr, hs.dev<float>(o_y), n_out, st);
  });
}
