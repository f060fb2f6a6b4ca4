// Pitch shifter: a peak-locked phase vocoder (Laroche & Dolson 1999) on the denoiser's STFT, fp32 on the device in every
// vtts_precision mode, with the phase recurrence in double:
//   STFT n_fft 1024 / hop 256 / periodic Hann / reflect padding 512 (F = n / 256 + 1 frames) | a = |X|, theta = arg X |
//   peaks: a[k] > a[k-1], a[k] >= a[k+1], a[k] > 0 (neighbours outside [0, 512] count as -1) | every bin belongs to its
//   nearest peak, the lower one on a tie | omega_t[p] = 2 pi p / N + princarg(theta_t[p] - theta_t-1[p] - 2 pi p H / N) / H
//   (2 pi p / N at t = 0) | psi_t(p) = princarg(psi_t-1[p] + H (r - 1) omega_t[p]), psi_t-1[k] the rotation of the peak
//   that owned bin k in frame t - 1 (0 before frame 0 and in a frame without peaks) | bin k of peak p moves to
//   k + D_p, D_p = rint((r - 1) p), times (-1)^D_p e^(i psi_t(p)), targets outside [0, 512] dropped, contributions summed
//   in ascending k | the denoiser's inverse and overlap-add.
// r = fp32(2^(s / 12)), s in [-12, 12].  Rows with s == 0, and rows of <= 512 samples, are copied.
//
// Analysis kernel.  One warp per frame, as denoise_frame_kernel: the frame is read and transformed ALONE, so its
// outputs (X, theta in double, the owner map) are a function of its own 1024 input samples.
// Phase kernel.  One CTA per row, one thread per bin, walks the row's frames in order: the only sequential part.  A peak
// thread computes its rotation into shared memory; after one barrier every bin takes its owner's.  Double buffering of
// the shared rotations makes that one barrier per frame.
// Synthesis kernel.  One warp per frame: the rotated bins and their targets go to shared memory, lane l then sums the
// targets [16 l, 16 l + 16) over the sources in ascending order, and the denoiser's inverse transform windows the frame.
// Overlap-add.  denoise_ola_kernel itself (vtts_denoise_ola).
//
// Stream.  Per slot the denoiser's window (2048 carried inputs plus one chunk), the 64-bit position, the next unscanned
// frame, theta and psi (double) of the last scanned frame, and the synthesized frames later outputs still overlap, in
// two halves that alternate per push (the carried frames are copied from the other half by the synthesis kernel).  A
// frame is scanned once it reads no input past the ones received (256 g + 512 <= P, and P > 512 for frame 0's
// reflection), or at END; outputs are released on the denoiser's schedule.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "stft_common.cuh"
#include "vtts_internal.cuh"

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
constexpr double TWO_PI = 6.283185307179586;

struct PsShift {
  float r;            // fp32(2^(s / 12))
  int copy;           // s == 0
};

struct PsRow {
  long long x0;       // absolute index of input buffer element 0
  long long n;        // row length (DN_OPEN while a stream slot is open)
  long long q0;       // first frame this call scans (analysis, phase step, synthesis)
  long long fb;       // first frame of the synthesized-frame buffer this call fills
  long long fb_prev;  // stream: first frame of the slot's other half; frames [fb, q0) are copied from it
  int nq;             // frames scanned
  int nsyn;           // frames of the buffer: [fb, fb + nsyn)
  int half;           // stream: the half of the slot's frame buffer this call fills
  int copy;           // the outputs are the inputs
  float r;            // ratio
  int pad_;
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
  r.copy = r.n <= PAD || shifts[b].copy;
  r.nq = r.copy ? 0 : (int)(r.n / HOP + 1);
  r.nsyn = r.nq;
  r.pad_ = 0;
  return r;
}

__device__ __forceinline__ double princarg(double x) { return x - TWO_PI * rint(x / TWO_PI); }

__global__ void __launch_bounds__(PS_WARPS * 32) pitch_analysis_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                      const int* __restrict__ n_in, const PsShift* __restrict__ shifts,
                                                                      const PsRow* __restrict__ rows, const float* __restrict__ hann,
                                                                      const float2* __restrict__ tw, PsWs w) {
  __shared__ float2 smem[PS_WARPS * 32 * TP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y, fl = blockIdx.x * PS_WARPS + warp;
  const PsRow r = ps_row(rows, n_in, shifts, S, b);
  if (fl >= r.nq) return;                                // warps are independent: no block-level barrier below
  float2* sw = smem + (size_t)warp * 32 * TP;
  float2 v[32];
  stftc::read_frame(v, x + (size_t)b * x_ld, r.x0, r.n, (r.q0 + fl) * HOP - PAD, hann, lane);
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
}

// state: stream [rows][2][513] (theta, psi of the last scanned frame) or nullptr; ola: one-shot, receives the rows'
// overlap-add bounds; dec: [rows][dec_fr][513] decisions, 1 | (e < 0) << 1 at a peak whose wrapped phase deviation is e,
// 0 elsewhere (test hook)
__global__ void __launch_bounds__(PH_THREADS) pitch_phase_kernel(const int* __restrict__ n_in, const PsShift* __restrict__ shifts,
                                                                const PsRow* __restrict__ rows, int S, PsWs w, double* __restrict__ state,
                                                                DnRow* __restrict__ ola, int* __restrict__ dec, int dec_fr) {
  __shared__ double ps_sh[2][NB];
  const int b = blockIdx.x, k = threadIdx.x;
  const PsRow r = ps_row(rows, n_in, shifts, S, b);
  if (ola && k == 0) {
    DnRow d;
    d.x0 = 0;
    d.n = r.n;
    d.g0 = 0;
    d.e0 = 0;
    d.cnt = S;
    d.nfr = r.nq;
    d.copy = r.copy;
    ola[b] = d;
  }
  if (r.nq == 0) return;                                 // uniform over the CTA
  const bool bin = k < NB;
  const double hr1 = HOP * ((double)r.r - 1.0);
  double thp = 0.0, psp = 0.0;
  if (state && bin) {
    thp = state[(size_t)b * 2 * NB + k];
    psp = state[(size_t)b * 2 * NB + NB + k];
  }
  const size_t f0 = (size_t)b * w.fr;
  int own = bin ? w.own[f0 * OWN_LD + k] : -1;
  double th = bin ? w.th[f0 * NB + k] : 0.0;
  for (int i = 0; i < r.nq; ++i) {
    const long long g = r.q0 + i;
    int own_n = -1;
    double th_n = 0.0;
    if (bin && i + 1 < r.nq) {                           // the next frame's loads fly under this frame's step
      own_n = w.own[(f0 + i + 1) * OWN_LD + k];
      th_n = w.th[(f0 + i + 1) * NB + k];
    }
    int neg = 0;
    if (own == k) {
      double om = TWO_PI * k / NF, prev = 0.0;
      if (g > 0) {
        const double e = princarg(th - thp - TWO_PI * k * HOP / NF);
        neg = e < 0.0;
        om += e / HOP;
        prev = psp;
      }
      ps_sh[i & 1][k] = princarg(prev + hr1 * om);
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
  }
  if (state && bin) {
    state[(size_t)b * 2 * NB + k] = thp;
    state[(size_t)b * 2 * NB + NB + k] = psp;
  }
}

__global__ void __launch_bounds__(PS_WARPS * 32) pitch_synth_kernel(const int* __restrict__ n_in, const PsShift* __restrict__ shifts,
                                                                   const PsRow* __restrict__ rows, int S, const float* __restrict__ hann,
                                                                   const float2* __restrict__ tw, PsWs w) {
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

int ps_check_shifts(vtts_ctx* ctx, const char* who, const float* semitones, int n) {
  if (!semitones) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null semitones", who);
  for (int i = 0; i < n; ++i)
    if (!shift_ok(semitones[i]))
      return ctx->fail(VTTS_ERR_BAD_ARG, "%s: semitones[%d] = %g (finite, in [-12, 12])", who, i, (double)semitones[i]);
  return VTTS_OK;
}

// fp32(2^(s / 12)), computed in double and rounded once
float ps_ratio(float s) { return (float)std::pow(2.0, (double)s / 12.0); }

void ps_carve(Arena& a, PsWs& w, int rows) {
  w.X = a.take<float2>((size_t)rows * w.fr * NB);
  w.th = a.take<double>((size_t)rows * w.fr * NB);
  w.own = a.take<short>((size_t)rows * w.fr * OWN_LD);
  w.psi = a.take<double>((size_t)rows * w.fr * NB);
  w.syn = a.take<float>((size_t)rows * w.halves * w.nbuf * NF);
}

// analysis, phase, synthesis (three launches); the synthesis is skipped when only the decisions are wanted
int ps_launch(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const PsShift* shifts, const PsRow* rows, int B,
              long long max_nq, long long max_nsyn, const PsWs& w, double* state, DnRow* ola, int* dec, int dec_fr, cudaStream_t st) {
  const float2* tw = reinterpret_cast<const float2*>(ctx->fft_tw);
  const unsigned agrid = (unsigned)std::max(1LL, (max_nq + PS_WARPS - 1) / PS_WARPS);
  pitch_analysis_kernel<<<dim3(agrid, B), PS_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, shifts, rows, ctx->hann, tw, w);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  pitch_phase_kernel<<<B, PH_THREADS, 0, st>>>(n_in, shifts, rows, S, w, state, ola, dec, dec_fr);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  if (dec) return VTTS_OK;
  const unsigned sgrid = (unsigned)std::max(1LL, (max_nsyn + PS_WARPS - 1) / PS_WARPS);
  pitch_synth_kernel<<<dim3(sgrid, B), PS_WARPS * 32, 0, st>>>(n_in, shifts, rows, S, ctx->hann, tw, w);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// one-shot call (dec == nullptr) or the decisions test hook
int ps_one_shot(vtts_ctx* ctx, const char* who, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, float* y_dev,
                int* dec_dev, cudaStream_t st) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!x_dev || !(y_dev || dec_dev)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: y must not alias x", who);
  if (B < 1 || B > 65535 || S < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: B=%d S=%d (1..65535, >= 1)", who, B, S);
  int rc = ps_check_shifts(ctx, who, semitones, B);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  const int F = S / HOP + 1;
  PsWs w{};
  w.fr = F;
  w.nbuf = F;
  w.halves = 1;
  Arena m(nullptr, 0, true);
  m.take<PsShift>(B);
  m.take<DnRow>(B);
  ps_carve(m, w, B);
  rc = ctx->ensure_ws(m.off);
  if (rc) return rc;
  Arena a(ctx->ws, ctx->ws_bytes, false);
  PsShift* shifts = a.take<PsShift>(B);
  DnRow* ola = a.take<DnRow>(B);
  ps_carve(a, w, B);
  std::vector<PsShift> h(B);
  for (int b = 0; b < B; ++b) h[b] = PsShift{ps_ratio(semitones[b]), semitones[b] == 0.f};
  // pageable source: the call returns once the table is staged
  VTTS_CUDA(cudaMemcpyAsync(shifts, h.data(), (size_t)B * sizeof(PsShift), cudaMemcpyHostToDevice, st));
  if (dec_dev) {
    VTTS_CUDA(cudaMemsetAsync(dec_dev, 0, (size_t)B * F * NB * sizeof(int), st));
    return ps_launch(ctx, x_dev, S, S, n_dev, shifts, nullptr, B, F, F, w, nullptr, nullptr, dec_dev, F, st);
  }
  rc = ps_launch(ctx, x_dev, S, S, n_dev, shifts, nullptr, B, F, F, w, nullptr, ola, nullptr, 0, st);
  if (rc) return rc;
  return vtts_denoise_ola(ctx, x_dev, S, S, nullptr, ola, B, S, w.syn, w.nbuf, y_dev, S, st);
}

}  // namespace

int vtts_pitch_shift_stream_lookahead(void) { return PS_LOOKAHEAD; }

int vtts_pitch_shift(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, float* y_dev,
                     void* stream) {
  if (ctx && !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift: null pointer");
  return ps_one_shot(ctx, "pitch_shift", x_dev, n_dev, B, S, semitones, y_dev, nullptr, (cudaStream_t)stream);
}

int vtts_debug_pitch_decisions(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, int32_t* dec_dev,
                               void* stream) {
  if (ctx && !dec_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_pitch_decisions: null pointer");
  return ps_one_shot(ctx, "debug_pitch_decisions", x_dev, n_dev, B, S, semitones, nullptr, dec_dev, (cudaStream_t)stream);
}

int vtts_pitch_shift_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* semitones, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!x || !y || B < 1 || B > 65535 || S < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_host: bad argument (B=%d S=%d)", B, S);
  int rc = ps_check_shifts(ctx, "pitch_shift_host", semitones, B);
  if (rc) return rc;
  if (n_in)
    for (int b = 0; b < B; ++b)
      if (n_in[b] < 0 || n_in[b] > S) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_host: n[%d]=%d outside [0, %d]", b, n_in[b], S);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)B * S * 4, n_b = (size_t)B * 4;
  const size_t o_n = (x_b + 255) & ~size_t(255), o_y = (o_n + n_b + 255) & ~size_t(255);
  rc = ctx->ensure_staging(o_y + x_b, o_y + x_b);
  if (rc) return rc;
  char* hp = (char*)ctx->hpin;
  char* dp = (char*)ctx->dstage;
  cudaStream_t st = ctx->own_stream;
  memcpy(hp, x, x_b);
  if (n_in) memcpy(hp + o_n, n_in, n_b);
  VTTS_CUDA(cudaMemcpyAsync(dp, hp, o_n + n_b, cudaMemcpyHostToDevice, st));
  rc = vtts_pitch_shift(ctx, (const float*)dp, n_in ? (const int32_t*)(dp + o_n) : nullptr, B, S, semitones, (float*)(dp + o_y), st);
  if (rc) {
    cudaStreamSynchronize(st);   // the staging copy must not outlive the call
    return rc;
  }
  VTTS_CUDA(cudaMemcpyAsync(hp + o_y, dp + o_y, x_b, cudaMemcpyDeviceToHost, st));
  VTTS_CUDA(cudaStreamSynchronize(st));
  memcpy(y, hp + o_y, x_b);
  return VTTS_OK;
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct vtts_pitch_shift_stream {
  vtts_ctx* ctx = nullptr;
  int S = 0, F = 0, cap = 0, out_pitch = 0;
  PsWs w{};
  void* mem = nullptr;          // windows [S][cap], the workspace, state [S][2][513], then the per-push tables
  float* win = nullptr;
  double* state = nullptr;
  DnRow* d_rows = nullptr;      // tables: DnRow [S], PsRow [S], int [S][2], one copy per push
  // per slot: inputs received since BEGIN, outputs emitted, next unscanned frame, first frame and half of the last
  // push's synthesized-frame buffer, open, inputs of the last push whose tail has not moved yet, shift since BEGIN
  std::vector<long long> P, E, q, fb;
  std::vector<int> open, pending, half;
  std::vector<float> semis;
  std::vector<char> tbl;        // host image of the per-push tables
};

int vtts_pitch_shift_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, vtts_pitch_shift_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!out || !out_pitch) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_create: null pointer");
  *out = nullptr;
  if (max_streams < 1 || max_streams > 65535 || max_chunk_samples < 1 || max_chunk_samples > (1 << 22))
    return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_create: max_streams=%d max_chunk_samples=%d (1..65535, 1..%d)", max_streams,
                     max_chunk_samples, 1 << 22);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  int rc = vtts_fft_tables(ctx);
  if (rc) return rc;
  vtts_pitch_shift_stream* ps = new vtts_pitch_shift_stream;
  const int S = max_streams;
  ps->ctx = ctx;
  ps->S = S;
  ps->F = max_chunk_samples;
  ps->cap = PS_K + max_chunk_samples;
  ps->out_pitch = max_chunk_samples + PS_LOOKAHEAD;    // as the denoise stream
  // frames scanned per push: at most n_new / 256 + 3 (with END); the buffer also holds the <= 3 carried frames
  ps->w.fr = max_chunk_samples / HOP + 4;
  ps->w.nbuf = ps->w.fr + 4;
  ps->w.halves = 2;
  const size_t tbl_b = (size_t)S * (sizeof(DnRow) + sizeof(PsRow) + 2 * sizeof(int));
  Arena m(nullptr, 0, true);
  m.take<float>((size_t)S * ps->cap);
  PsWs w = ps->w;
  ps_carve(m, w, S);
  m.take<double>((size_t)S * 2 * NB);
  m.take<char>(tbl_b);
  const size_t bytes = m.off;
  cudaError_t e = cudaMalloc(&ps->mem, bytes);
  if (e == cudaSuccess) e = cudaMemset(ps->mem, 0, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (ps->mem) cudaFree(ps->mem);
    delete ps;
    return ctx->fail(e == cudaErrorMemoryAllocation ? VTTS_ERR_OOM : VTTS_ERR_CUDA, "pitch_shift_stream_create: %zu bytes: %s", bytes,
                     cudaGetErrorString(e));
  }
  Arena a(ps->mem, bytes, false);
  ps->win = a.take<float>((size_t)S * ps->cap);
  ps_carve(a, ps->w, S);
  ps->state = a.take<double>((size_t)S * 2 * NB);
  ps->d_rows = reinterpret_cast<DnRow*>(a.take<char>(tbl_b));
  ps->P.assign(S, 0);
  ps->E.assign(S, 0);
  ps->q.assign(S, 0);
  ps->fb.assign(S, 0);
  ps->open.assign(S, 0);
  ps->pending.assign(S, 0);
  ps->half.assign(S, 0);
  ps->semis.assign(S, 0.f);
  ps->tbl.assign(tbl_b, 0);
  *out = ps;
  *out_pitch = ps->out_pitch;
  return VTTS_OK;
}

int vtts_pitch_shift_stream_destroy(vtts_ctx* ctx, vtts_pitch_shift_stream* ps) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!ps) return VTTS_OK;
  if (ps->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_destroy: the stream belongs to another context");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());   // a push may still be running on the caller's stream
  cudaFree(ps->mem);
  delete ps;
  return VTTS_OK;
}

int vtts_pitch_shift_stream_push(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                 const float* semitones, float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!ps || ps->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: the stream belongs to another context");
  if (!x_dev || !n_new || !flags || !y_dev || !n_out) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: null pointer");
  if (x_dev == y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: y must not alias x");
  const int S = ps->S, F = ps->F;
  for (int s = 0; s < S; ++s) {
    if (n_new[s] < 0 || n_new[s] > F)
      return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: n_new[%d]=%d outside [0, %d]", s, n_new[s], F);
    if (flags[s] & ~3u) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: flags[%d]=%u (bit0 BEGIN, bit1 END)", s, flags[s]);
    const bool idle = n_new[s] == 0 && flags[s] == 0;
    if (idle) continue;
    if (!(flags[s] & 1) && !ps->open[s])
      return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: slot %d is not open (push BEGIN first, also after END)", s);
    if (flags[s] & 1) {
      if (!semitones) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: BEGIN needs the semitones array");
      if (!shift_ok(semitones[s]))
        return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: semitones[%d] = %g (finite, in [-12, 12])", s, (double)semitones[s]);
    } else if (semitones && !(semitones[s] == ps->semis[s])) {
      return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push: semitones[%d] = %g, but slot %d shifts by %g until END (BEGIN to change it)",
                       s, (double)semitones[s], s, (double)ps->semis[s]);
    }
  }
  VTTS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;

  // ---- host bookkeeping: outputs [E0, E1), frames [q0, q1) scanned, synthesized-frame buffer [fb, q1) ----
  DnRow* rows = reinterpret_cast<DnRow*>(ps->tbl.data());
  PsRow* prow = reinterpret_cast<PsRow*>(ps->tbl.data() + (size_t)S * sizeof(DnRow));
  int* prep = reinterpret_cast<int*>(ps->tbl.data() + (size_t)S * (sizeof(DnRow) + sizeof(PsRow)));
  std::vector<long long> E1(S), Q1(S);
  long long max_out = 0, max_nq = 0, max_nsyn = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = n_new[s] > 0 || flags[s] != 0, begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : ps->P[s], E0 = begin ? 0 : ps->E[s], P1 = P0 + n_new[s];
    const float sm = begin ? semitones[s] : ps->semis[s];
    long long e = E0;
    if (act) e = end ? P1 : std::min(P1, (long long)HOP * std::max(0LL, P1 / HOP - 3));
    E1[s] = e;
    n_out[s] = (int32_t)(e - E0);
    DnRow r{};
    PsRow p{};
    r.x0 = p.x0 = P0 - PS_K;
    r.n = p.n = end ? P1 : DN_OPEN;
    r.e0 = E0;
    r.cnt = e - E0;
    r.copy = p.copy = sm == 0.f || (end && P1 <= PAD);
    p.r = ps_ratio(sm);
    const long long q0 = begin ? 0 : ps->q[s];
    Q1[s] = q0;
    if (act && !p.copy) {
      const long long q1 = end ? P1 / HOP + 1 : (P1 > PAD ? (P1 - PAD) / HOP + 1 : 0);
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
        return ctx->fail(VTTS_ERR_CUDA, "pitch_shift_stream_push: slot %d frames [%lld, %lld) buffer from %lld (internal bound %d / %d)", s, q0,
                         q1, fb, ps->w.fr, ps->w.nbuf);
    }
    if (r.cnt > ps->out_pitch)
      return ctx->fail(VTTS_ERR_CUDA, "pitch_shift_stream_push: slot %d needs %lld outputs (internal bound %d)", s, r.cnt, ps->out_pitch);
    rows[s] = r;
    prow[s] = p;
    prep[2 * s] = act && !begin ? ps->pending[s] : 0;
    prep[2 * s + 1] = act ? n_new[s] : 0;
    max_out = std::max(max_out, r.cnt);
    max_nq = std::max(max_nq, (long long)p.nq);
    max_nsyn = std::max(max_nsyn, (long long)p.nsyn);
  }

  // ---- device: table copy, window step, analysis, phase, synthesis, overlap-add (five launches) ----
  // pageable source: the call returns once the table is staged, so ps->tbl may be rewritten by the next push
  VTTS_CUDA(cudaMemcpyAsync(ps->d_rows, ps->tbl.data(), ps->tbl.size(), cudaMemcpyHostToDevice, st));
  const PsRow* d_prow = reinterpret_cast<const PsRow*>(reinterpret_cast<const char*>(ps->d_rows) + (size_t)S * sizeof(DnRow));
  const int* d_prep = reinterpret_cast<const int*>(reinterpret_cast<const char*>(ps->d_rows) + (size_t)S * (sizeof(DnRow) + sizeof(PsRow)));
  int rc = vtts_stream_window_prep(ctx, ps->win, ps->cap, PS_K, d_prep, x_dev, F, S, st);
  if (rc) return rc;
  rc = ps_launch(ctx, ps->win, ps->cap, ps->cap, nullptr, nullptr, d_prow, S, max_nq, max_nsyn, ps->w, ps->state, nullptr, nullptr, 0, st);
  if (rc) return rc;
  rc = vtts_denoise_ola(ctx, ps->win, ps->cap, ps->cap, nullptr, ps->d_rows, S, max_out, ps->w.syn, 2 * ps->w.nbuf, y_dev, ps->out_pitch,
                        st);
  if (rc) return rc;

  // ---- commit the slot state ----
  for (int s = 0; s < S; ++s) {
    const bool act = n_new[s] > 0 || flags[s] != 0, begin = flags[s] & 1, end = flags[s] & 2;
    if (!act) continue;
    if (begin) ps->semis[s] = semitones[s];
    if (prow[s].nsyn > 0 || prow[s].nq > 0) {
      ps->fb[s] = prow[s].fb;
      ps->half[s] = prow[s].half;
    } else if (begin) {
      ps->fb[s] = 0;
      ps->half[s] = 0;
    }
    ps->q[s] = Q1[s];
    ps->P[s] = (begin ? 0 : ps->P[s]) + n_new[s];
    ps->E[s] = E1[s];
    ps->open[s] = !end;
    ps->pending[s] = end ? 0 : n_new[s];
  }
  return VTTS_OK;
}

int vtts_pitch_shift_stream_push_host(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x, const int32_t* n_new, const uint8_t* flags,
                                      const float* semitones, float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!ps || ps->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push_host: the stream belongs to another context");
  if (!x || !y) return ctx->fail(VTTS_ERR_BAD_ARG, "pitch_shift_stream_push_host: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)ps->S * ps->F * 4, y_b = (size_t)ps->S * ps->out_pitch * 4;
  const size_t o_y = (x_b + 255) & ~size_t(255);
  int rc = ctx->ensure_staging(o_y + y_b, o_y + y_b);
  if (rc) return rc;
  char* hp = (char*)ctx->hpin;
  char* dp = (char*)ctx->dstage;
  cudaStream_t st = ctx->own_stream;
  memcpy(hp, x, x_b);
  VTTS_CUDA(cudaMemcpyAsync(dp, hp, x_b, cudaMemcpyHostToDevice, st));
  rc = vtts_pitch_shift_stream_push(ctx, ps, (const float*)dp, n_new, flags, semitones, (float*)(dp + o_y), n_out, st);
  if (rc) {
    cudaStreamSynchronize(st);   // the staging copy must not outlive the call
    return rc;
  }
  VTTS_CUDA(cudaMemcpyAsync(hp + o_y, dp + o_y, y_b, cudaMemcpyDeviceToHost, st));
  VTTS_CUDA(cudaStreamSynchronize(st));
  memcpy(y, hp + o_y, y_b);
  return VTTS_OK;
}
