// Lookahead true-peak limiter of one mono row, fp32 on the device in every vtts_precision mode (oracle/limiter_oracle.py
// states it in float64):
//   v = fp32(10^(G / 20)) x;  u = resample_poly(v, 4, 1) (the loudness meter's true-peak oversampler, vtts_resample_run);
//   p[t] = max(|v[t]|, max |u[j]| over j in [4(t - D), 4(t + D) + 3] inside [0, 4n)), D = 10;  tau = min(1, c / p)
//   (1 where p = 0 and past the row's end);  hold h[t] = min tau[t .. t + W - 1];  attack a[t] = the mean of
//   q = ceil((1 - h) 2^32) over [t - W + 1, t] (q = 0 before sample 0), rounded up, times 2^-32;  release
//   d[t] = max(a_t, beta d[t - 1] + (1 - beta) a_t);  y = v min(tau, 1 - d);  reduction = 20 log10 min(applied gain).
//
// Invariant.  As in loudness.cu, every value is a fixed fp32 function of the samples and of state carried at
// boundaries fixed by absolute sample index: tau and a read fixed neighbourhoods (min and integer sums give the same
// bits in any order), and the release runs as a scan of the monotone maps f_t(d) = max(a_t, fma(beta, d, e_t)),
// e_t = fp32(1 - beta) a_t.  Their compositions keep the form M(d) = max(c, fma(m, d, k)): f_t after M is
// (max(a_t, fma(beta, c, e_t)), beta m, fma(beta, k, e_t)), the identity (-inf, 1, 0).  The maps are folded in sample
// order over blocks of Q = 256 samples fixed by absolute index (fold kernel, one thread per block), chained over the
// blocks by one thread per row (d_in of block i + 1 = M_i(d_in of block i), from d = 0), and refolded per block while
// d[t] = M_<=t(d_in) is evaluated at every sample (apply kernel).  A row therefore gives the same bits alone, in any
// batch position, in every precision mode, and through the stream at any push pattern.
//
// Stream.  Per slot a window of H = 2W + 64 carried samples plus one chunk (the resample stream's window step), the
// partial map of the block holding the next output, that block's d_in, and the running minimum gain.  Sample t is
// released once sample t + W + D + 9 has arrived (the last input tau[t + W - 1] reads through the oversampler);
// END releases the rest.  Every push issues the same nine launches.
#include <algorithm>
#include <cmath>

#include "stream_common.cuh"

namespace {

constexpr int D = 10;                 // p[t] reads u over t +- D input samples
constexpr int OS = 4;                 // true-peak oversampling
constexpr int Q = 256;                // block of the release scan
constexpr int TILE = 1024;            // samples per CTA of the tau and hold / attack kernels
constexpr int THREADS = 256;
constexpr int SCAN_THREADS = 128;     // fold / chain / apply / finish: one thread per block or row
constexpr int W_MAX = 3840;           // rint(20 ms * 192 kHz)
constexpr unsigned FULL = 0xffffffffu;

struct LmRow {
  long long x0;      // absolute index of element 0 of the row's v / tau / a buffers
  long long u0;      // absolute index of element 0 of the row's u buffer
  long long n;       // row length (a stream slot before END: the samples received)
  long long ta, tn;  // tau is computed for samples [ta, ta + tn)
  long long r0, rn;  // the outputs: samples [r0, r0 + rn), y element 0 = r0
  float gain_db;
  int begin;         // the carried release state restarts
};
static_assert(sizeof(LmRow) % 16 == 0, "table entries keep 16-byte alignment");

// rows == nullptr: the one-shot row b, n = n_in[b] clamped to [0, S], gain gdb[b] (or 0 dB)
__device__ __forceinline__ LmRow lm_row(const LmRow* rows, const int* n_in, const float* gdb, int S, int b) {
  if (rows) return rows[b];
  LmRow r;
  r.n = n_in ? min(max(n_in[b], 0), S) : S;
  r.x0 = r.u0 = 0;
  r.ta = r.r0 = 0;
  r.tn = r.rn = r.n;
  r.gain_db = gdb ? gdb[b] : 0.f;
  r.begin = 1;
  return r;
}

__device__ __forceinline__ int lm_blocks(const LmRow& r) { return r.rn > 0 ? (int)((r.r0 + r.rn - 1) / Q - r.r0 / Q + 1) : 0; }

// v element e = sample x0 + e times fp32(10^(G / 20)) (G clamped to [-70, 70], 0 if not finite) inside [0, n), else 0;
// y_zero (one-shot): y[t] = 0 for t in [n, S) (y may be x: only samples past n are written)
__global__ void __launch_bounds__(THREADS) lm_gain_kernel(const float* x, long long x_ld, int S, const int* __restrict__ n_in,
                                                          const float* __restrict__ gdb, const LmRow* __restrict__ rows, long long vn,
                                                          float* __restrict__ v, long long v_ld, float* y_zero) {
  const int b = blockIdx.y;
  const long long e = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (e >= vn) return;
  const LmRow r = lm_row(rows, n_in, gdb, S, b);
  float g = r.gain_db;
  g = isfinite(g) ? fminf(fmaxf(g, -70.f), 70.f) : 0.f;
  const float f = (float)exp10((double)g / 20.0);
  const long long t = r.x0 + e;
  const bool in = t >= 0 && t < r.n;
  v[(size_t)b * v_ld + e] = in ? x[(size_t)b * x_ld + e] * f : 0.f;
  if (y_zero && !in) y_zero[(size_t)b * x_ld + e] = 0.f;
}

// tau over samples [ta, ta + tn): a CTA stages gm[k] = max |u[4k .. 4k + 3]| (inside [0, 4n)) for its tile +- D
__global__ void __launch_bounds__(THREADS) lm_tau_kernel(const float* __restrict__ v, long long v_ld, const float* __restrict__ u,
                                                         long long u_ld, int S, const int* __restrict__ n_in,
                                                         const LmRow* __restrict__ rows, float c, float* __restrict__ tau) {
  __shared__ float gm[TILE + 2 * D];
  const int b = blockIdx.y;
  const LmRow r = lm_row(rows, n_in, nullptr, S, b);
  const long long tA = r.ta + (long long)blockIdx.x * TILE;
  if (tA >= r.ta + r.tn) return;
  const int cnt = (int)min((long long)TILE, r.ta + r.tn - tA);
  const float* ur = u + (size_t)b * u_ld;
  for (int i = threadIdx.x; i < cnt + 2 * D; i += THREADS) {
    const long long k = tA - D + i;
    float m = 0.f;
    if (k >= 0 && k < r.n) {
      const float* q = ur + (OS * k - r.u0);
#pragma unroll
      for (int o = 0; o < OS; ++o) m = fmaxf(m, fabsf(__ldg(q + o)));
    }
    gm[i] = m;
  }
  __syncthreads();
  const float* vr = v + (size_t)b * v_ld - r.x0;
  float* tr = tau + (size_t)b * v_ld - r.x0;
  for (int i = threadIdx.x; i < cnt; i += THREADS) {
    const long long t = tA + i;
    float p = fabsf(vr[t]);
#pragma unroll
    for (int o = 0; o <= 2 * D; ++o) p = fmaxf(p, gm[i + o]);
    tr[t] = (t < r.n && p > 0.f) ? fminf(1.f, c / p) : 1.f;
  }
}

size_t hold_smem(int W) {
  const size_t L1 = TILE + 2 * (size_t)W - 2, L2 = TILE + (size_t)W - 1;
  return 2 * L1 * sizeof(float) + L2 * sizeof(unsigned long long) + 64;
}

// a over samples [r0, r0 + rn).  A CTA stages tau over [A - W + 1, A + cnt + W - 1) (1 outside [0, n)), takes the
// sliding minimum h over [A - W + 1, A + cnt) by doubling (min over [i, i + 2^j), then two overlapping windows),
// quantizes q = 2^32 - floor(h 2^32) (0 before sample 0), scans q as 64-bit integers and takes the box differences.
__global__ void __launch_bounds__(THREADS) lm_attack_kernel(const float* __restrict__ tau, long long v_ld, int S,
                                                            const int* __restrict__ n_in, const LmRow* __restrict__ rows, int W,
                                                            float* __restrict__ alpha) {
  extern __shared__ __align__(16) unsigned char lm_smem[];
  const int b = blockIdx.y, tid = threadIdx.x;
  const LmRow r = lm_row(rows, n_in, nullptr, S, b);
  const long long A = r.r0 + (long long)blockIdx.x * TILE;
  if (A >= r.r0 + r.rn) return;
  const int cnt = (int)min((long long)TILE, r.r0 + r.rn - A);
  const int L1 = cnt + 2 * W - 2, L2 = cnt + W - 1;
  unsigned long long* qs = reinterpret_cast<unsigned long long*>(lm_smem);
  float* s0 = reinterpret_cast<float*>(qs + (TILE + W));
  float* s1 = s0 + (TILE + 2 * W);
  const long long base = A - W + 1;
  const float* tr = tau + (size_t)b * v_ld - r.x0;
  for (int i = tid; i < L1; i += THREADS) {
    const long long t = base + i;
    s0[i] = (t >= 0 && t < r.n) ? tr[t] : 1.f;
  }
  __syncthreads();
  int w = 1;
  while (2 * w <= W) {                      // s0[i] = min over [i, i + 2w)
    for (int i = tid; i < L1 - w; i += THREADS) s1[i] = fminf(s0[i], s0[i + w]);
    __syncthreads();
    for (int i = tid; i < L1 - w; i += THREADS) s0[i] = s1[i];
    __syncthreads();
    w *= 2;
  }
  const int partial = W - w;                // h[i] = min(s0[i], s0[i + W - w])
  // per thread a contiguous run of q, summed, then a block scan of the run totals
  const int run = (L2 + THREADS - 1) / THREADS, i0 = min(tid * run, L2), i1 = min(i0 + run, L2);
  unsigned long long tot = 0;
  for (int i = i0; i < i1; ++i) {
    const float h = fminf(s0[i], s0[i + partial]);
    const unsigned long long q = base + i < 0 ? 0ull : (1ull << 32) - (unsigned long long)(h * 4294967296.f);
    tot += q;
    qs[i] = tot;
  }
  // exclusive scan of tot over the CTA
  const int lane = tid & 31, warp = tid >> 5;
  unsigned long long incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(FULL, incl, o);
    if (lane >= o) incl += y;
  }
  __shared__ unsigned long long wsum[THREADS / 32];
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  unsigned long long off = incl - tot;
  for (int k = 0; k < warp; ++k) off += wsum[k];
  for (int i = i0; i < i1; ++i) qs[i] += off;
  __syncthreads();
  float* ar = alpha + (size_t)b * v_ld - r.x0;
  for (int o = tid; o < cnt; o += THREADS) {
    const unsigned long long sum = qs[o + W - 1] - (o > 0 ? qs[o - 1] : 0ull);
    const unsigned long long qa = (sum + (unsigned long long)W - 1) / (unsigned long long)W;
    ar[A + o] = __ull2float_ru(qa) * 2.3283064365386963e-10f;   // 2^-32
  }
}

// the release maps (Map, map_fold, map_apply) live in vtts_internal.cuh, shared with the compressor

// the samples [lo, hi) of call block i of row r
__device__ __forceinline__ void lm_block_span(const LmRow& r, int i, long long& lo, long long& hi) {
  const long long kb = r.r0 / Q + i;
  lo = max(r.r0, kb * Q);
  hi = min(r.r0 + r.rn, (kb + 1) * Q);
}

// maps[row][i] = the fold of call block i, from the carried partial map for i = 0 (stream rows that do not begin), else
// from the identity; start[row] = block 0's starting map
__global__ void __launch_bounds__(SCAN_THREADS) lm_fold_kernel(const float* __restrict__ alpha, long long v_ld, int S,
                                                               const int* __restrict__ n_in, const LmRow* __restrict__ rows,
                                                               float beta, float omb, const float4* __restrict__ carry_map,
                                                               float4* __restrict__ maps, int ld_blk, float4* __restrict__ start) {
  const int b = blockIdx.y, i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  const LmRow r = lm_row(rows, n_in, nullptr, S, b);
  if (i >= lm_blocks(r)) return;
  Map M = map_id();
  if (i == 0) {
    if (carry_map && !r.begin) {
      const float4 cm = carry_map[b];
      M = Map{cm.x, cm.y, cm.z};
    }
    start[b] = make_float4(M.c, M.m, M.k, 0.f);
  }
  long long lo, hi;
  lm_block_span(r, i, lo, hi);
  const float* ar = alpha + (size_t)b * v_ld - r.x0;
  for (long long t = lo; t < hi; ++t) map_fold(M, ar[t], beta, omb);
  maps[(size_t)b * ld_blk + i] = make_float4(M.c, M.m, M.k, 0.f);
}

// d_in[row][i] of every call block: the chain d <- M_i(d) over the blocks that end at a block boundary, from the carried
// d_in (0 when the row begins); the carry takes the d_in and partial map of the block holding the row's next output
__global__ void __launch_bounds__(SCAN_THREADS) lm_chain_kernel(int S, const int* __restrict__ n_in, const LmRow* __restrict__ rows, int B,
                                                                const float4* __restrict__ maps, int ld_blk, float* __restrict__ din,
                                                                float* carry_din, float4* carry_map) {
  const int b = blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (b >= B) return;
  const LmRow r = lm_row(rows, n_in, nullptr, S, b);
  const int nb = lm_blocks(r);
  float d = (carry_din && !r.begin) ? carry_din[b] : 0.f;
  float4 part = make_float4(-INFINITY, 1.f, 0.f, 0.f);
  if (carry_map && !r.begin) part = carry_map[b];
  for (int i = 0; i < nb; ++i) {
    din[(size_t)b * ld_blk + i] = d;
    long long lo, hi;
    lm_block_span(r, i, lo, hi);
    const float4 M = maps[(size_t)b * ld_blk + i];
    if (hi % Q == 0) {
      d = map_apply(Map{M.x, M.y, M.z}, d);
      part = make_float4(-INFINITY, 1.f, 0.f, 0.f);
    } else {
      part = M;
    }
  }
  if (carry_din) {
    carry_din[b] = d;
    carry_map[b] = part;
  }
}

// y[t] = v[t] min(tau[t], 1 - d[t]) over call block i, d[t] from the block's refold; gmin[row][i] = its least gain
__global__ void __launch_bounds__(SCAN_THREADS) lm_apply_kernel(const float* __restrict__ v, const float* __restrict__ tau,
                                                                const float* __restrict__ alpha, long long v_ld, int S,
                                                                const int* __restrict__ n_in, const LmRow* __restrict__ rows,
                                                                float beta, float omb, const float4* __restrict__ start,
                                                                const float* __restrict__ din, int ld_blk, float* y, long long y_ld,
                                                                float* __restrict__ gmin) {
  const int b = blockIdx.y, i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  const LmRow r = lm_row(rows, n_in, nullptr, S, b);
  if (i >= lm_blocks(r)) return;
  Map M = map_id();
  if (i == 0) {
    const float4 s = start[b];
    M = Map{s.x, s.y, s.z};
  }
  const float d0 = din[(size_t)b * ld_blk + i];
  long long lo, hi;
  lm_block_span(r, i, lo, hi);
  const size_t ro = (size_t)b * v_ld;
  const float *vr = v + ro - r.x0, *tr = tau + ro - r.x0, *ar = alpha + ro - r.x0;
  float* yr = y + (size_t)b * y_ld - r.r0;
  float gm = 1.f;
  for (long long t = lo; t < hi; ++t) {
    map_fold(M, ar[t], beta, omb);
    const float g = fminf(tr[t], 1.f - map_apply(M, d0));
    yr[t] = vr[t] * g;
    gm = fminf(gm, g);
  }
  gmin[(size_t)b * ld_blk + i] = gm;
}

// red[row] = 20 log10 of the least gain over the call's blocks and the carried minimum (stream rows that do not begin)
__global__ void __launch_bounds__(SCAN_THREADS) lm_finish_kernel(int S, const int* __restrict__ n_in, const LmRow* __restrict__ rows,
                                                                 int B, const float* __restrict__ gmin, int ld_blk,
                                                                 float* carry_min, float* __restrict__ red) {
  const int b = blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (b >= B) return;
  const LmRow r = lm_row(rows, n_in, nullptr, S, b);
  float g = (carry_min && !r.begin) ? carry_min[b] : 1.f;
  const int nb = lm_blocks(r);
  for (int i = 0; i < nb; ++i) g = fminf(g, gmin[(size_t)b * ld_blk + i]);
  if (carry_min) carry_min[b] = g;
  if (red) red[b] = 20.f * log10f(g);
}

// normalization gains: first = true: g = clamp(target - L) (0 where L = -inf); else g += target - L (unchanged where
// L = -inf), clamped to [-70, 70]
__global__ void lm_norm_gain_kernel(const float* __restrict__ readings, int B, float target, bool first, float* g) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float L = readings[b * 4];
  const float g0 = first ? 0.f : g[b];
  g[b] = isfinite(L) ? fminf(fmaxf(g0 + (target - L), -70.f), 70.f) : g0;
}

bool rate_ok(int rate) { return rate >= 8000 && rate <= 192000 && rate % 10 == 0; }

struct LmParams {
  int W;
  float beta, omb, c;
};

int lm_params(vtts_ctx* ctx, const char* who, int rate, float ceiling, float lookahead_ms, float release_ms, LmParams* p) {
  if (!rate_ok(rate)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rate %d (a multiple of 10 in [8000, 192000])", who, rate);
  if (!(ceiling >= -20.f && ceiling <= 0.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: ceiling %g dBTP (in [-20, 0])", who, (double)ceiling);
  if (!(lookahead_ms >= 1.f && lookahead_ms <= 20.f))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: lookahead %g ms (in [1, 20])", who, (double)lookahead_ms);
  if (!(release_ms >= 1.f && release_ms <= 2000.f))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: release %g ms (in [1, 2000])", who, (double)release_ms);
  p->W = std::max(1, (int)std::rint((double)lookahead_ms * rate / 1000.0));
  const double beta = std::exp(-1000.0 / ((double)release_ms * rate));
  p->beta = (float)beta;
  p->omb = (float)(1.0 - beta);
  p->c = (float)std::pow(10.0, (double)ceiling / 20.0);
  return VTTS_OK;
}

// the oversampled index S * OS of a one-shot row must fit an int
constexpr long long S_MAX = INT_MAX / OS;

// the parameters and batch shape of a one-shot call of entry point `who`
int lm_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, float ceiling, float lookahead_ms, float release_ms, LmParams* p) {
  const int rc = lm_params(ctx, who, rate, ceiling, lookahead_ms, release_ms, p);
  return rc ? rc : batch_check(ctx, who, B, S, S_MAX);
}

size_t al(size_t b) { return (b + 255) & ~size_t(255); }

// the buffers of one call: v, tau, alpha [rows][v_ld]; u [rows][u_ld]; per call block maps, d_in, least gain
struct LmBufs {
  float *v, *u, *tau, *alpha, *din, *gmin;
  float4 *maps, *start;
  long long v_ld, u_ld;
  int ld_blk;
  float4* carry_map;     // stream: [rows] carried partial map, else null
  float* carry_din;      // stream: [rows] carried d_in, else null
  float* carry_min;      // stream: [rows] running least gain, else null
};

int lm_blocks_max(long long rn) { return (int)(rn / Q + 2); }

size_t lm_oneshot_bytes(int B, int S) {
  const size_t nb = lm_blocks_max(S);
  return 3 * al((size_t)B * S * 4) + al((size_t)B * OS * S * 4) + al((size_t)B * nb * 16) + 2 * al((size_t)B * nb * 4) + al((size_t)B * 16);
}

void lm_oneshot_carve(void* ws, int B, int S, LmBufs* w) {
  Arena a(ws, SIZE_MAX, false);
  const size_t nb = lm_blocks_max(S);
  w->v = a.take<float>((size_t)B * S);
  w->tau = a.take<float>((size_t)B * S);
  w->alpha = a.take<float>((size_t)B * S);
  w->u = a.take<float>((size_t)B * OS * S);
  w->maps = a.take<float4>((size_t)B * nb);
  w->din = a.take<float>((size_t)B * nb);
  w->gmin = a.take<float>((size_t)B * nb);
  w->start = a.take<float4>(B);
  w->v_ld = S;
  w->u_ld = (long long)OS * S;
  w->ld_blk = (int)nb;
  w->carry_map = nullptr;
  w->carry_din = nullptr;
  w->carry_min = nullptr;
}

// the limiter's launches after v: the oversampler, tau, hold / attack, fold, chain, apply, finish
int lm_run(vtts_ctx* ctx, const LmParams& p, int rate, int S, const int* n_in, const LmRow* rows, const RsRow* rs_rows, int B,
           long long max_u, long long max_tn, long long max_rn, const LmBufs& w, float* y, long long y_ld, float* red, cudaStream_t st) {
  (void)rate;
  int rc = vtts_resample_run(ctx, 1, OS, w.v, w.v_ld, (int)w.v_ld, n_in, rs_rows, B, (long long)OS * S, max_u, w.u, w.u_ld, st);
  if (rc) return rc;
  lm_tau_kernel<<<dim3((unsigned)std::max(1LL, (max_tn + TILE - 1) / TILE), B), THREADS, 0, st>>>(w.v, w.v_ld, w.u, w.u_ld, S, n_in, rows,
                                                                                                  p.c, w.tau);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  static bool attr_set[64] = {};
  if (ctx->device < 64 && !attr_set[ctx->device]) {
    VTTS_CUDA(cudaFuncSetAttribute(lm_attack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hold_smem(W_MAX)));
    attr_set[ctx->device] = true;
  }
  const unsigned rtiles = (unsigned)std::max(1LL, (max_rn + TILE - 1) / TILE);
  lm_attack_kernel<<<dim3(rtiles, B), THREADS, hold_smem(p.W), st>>>(w.tau, w.v_ld, S, n_in, rows, p.W, w.alpha);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  const dim3 bgrid((unsigned)std::max(1, (lm_blocks_max(max_rn) + SCAN_THREADS - 1) / SCAN_THREADS), B);
  lm_fold_kernel<<<bgrid, SCAN_THREADS, 0, st>>>(w.alpha, w.v_ld, S, n_in, rows, p.beta, p.omb, w.carry_map, w.maps, w.ld_blk, w.start);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  const unsigned rgrid = (unsigned)((B + SCAN_THREADS - 1) / SCAN_THREADS);
  lm_chain_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.maps, w.ld_blk, w.din, w.carry_din, w.carry_map);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  lm_apply_kernel<<<bgrid, SCAN_THREADS, 0, st>>>(w.v, w.tau, w.alpha, w.v_ld, S, n_in, rows, p.beta, p.omb, w.start, w.din, w.ld_blk, y, y_ld,
                                                  w.gmin);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  lm_finish_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.gmin, w.ld_blk, w.carry_min, red);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// the one-shot limiter in the workspace at ws (sized by lm_oneshot_bytes)
int lm_oneshot(vtts_ctx* ctx, void* ws, const LmParams& p, int rate, const float* x, const int* n_in, const float* gain_db, int B, int S,
               float* y, float* red, cudaStream_t st) {
  LmBufs w;
  lm_oneshot_carve(ws, B, S, &w);
  lm_gain_kernel<<<dim3((S + THREADS - 1) / THREADS, B), THREADS, 0, st>>>(x, S, S, n_in, gain_db, nullptr, S, w.v, w.v_ld, y);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return lm_run(ctx, p, rate, S, n_in, nullptr, nullptr, B, (long long)OS * S, S, S, w, y, S, red, st);
}

// the one-shot limiter in the context workspace
int lm_launch(vtts_ctx* ctx, const LmParams& p, int rate, const float* x, const int* n_in, const float* gain_db, int B, int S, float* y, float* red,
              cudaStream_t st) {
  const int rc = ctx->ensure_ws(lm_oneshot_bytes(B, S));
  return rc ? rc : lm_oneshot(ctx, ctx->ws, p, rate, x, n_in, gain_db, B, S, y, red, st);
}

// the normalizer and limiter of a loudness_normalize_limited call whose arguments hold
int lnl_launch(vtts_ctx* ctx, const LmParams& p, const float* x, const int32_t* n_in, int B, int S, int rate, float target, float* y,
               float* gain_db, cudaStream_t st) {
  // the meter and the limiter each use the workspace from its start; the first pass's output, the readings and the
  // gains live past both
  const size_t front = al(std::max(vtts_loudness_ws_bytes(B, S, rate), lm_oneshot_bytes(B, S)));
  const size_t y1_b = al((size_t)B * S * 4), rd_b = al((size_t)B * 16);
  int rc = ctx->ensure_ws(front + y1_b + rd_b + al((size_t)B * 4));
  if (rc) return rc;
  char* base = (char*)ctx->ws;
  float* y1 = (float*)(base + front);
  float* rd = (float*)(base + front + y1_b);
  float* g = gain_db ? gain_db : (float*)(base + front + y1_b + rd_b);
  const unsigned gg = (unsigned)((B + 127) / 128);
  rc = vtts_loudness_launch(ctx, x, n_in, B, S, rate, rd, st);
  if (rc) return rc;
  lm_norm_gain_kernel<<<gg, 128, 0, st>>>(rd, B, target, true, g);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  rc = lm_oneshot(ctx, base, p, rate, x, n_in, g, B, S, y1, nullptr, st);
  if (!rc) rc = vtts_loudness_launch(ctx, y1, n_in, B, S, rate, rd, st);
  if (rc) return rc;
  lm_norm_gain_kernel<<<gg, 128, 0, st>>>(rd, B, target, false, g);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return lm_oneshot(ctx, base, p, rate, x, n_in, g, B, S, y, nullptr, st);
}

int lnl_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, float target, float ceiling, float lookahead_ms, float release_ms,
             LmParams* p) {
  const int rc = lm_args(ctx, who, B, S, rate, ceiling, lookahead_ms, release_ms, p);
  if (rc) return rc;
  if (!(target >= -70.f && target <= 0.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: target %g LUFS (in [-70, 0])", who, (double)target);
  return VTTS_OK;
}

}  // namespace

int vtts_limit(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, const float* gain_db_dev, int B, int S, int rate, float ceiling,
               float lookahead_ms, float release_ms, float* y_dev, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  LmParams p;
  const int rc = lm_args(ctx, "limit", B, S, rate, ceiling, lookahead_ms, release_ms, &p);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "limit: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return lm_launch(ctx, p, rate, x_dev, n_dev, gain_db_dev, B, S, y_dev, reduction_db_dev, (cudaStream_t)stream);
}

int vtts_limit_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, const float* gain_db, int B, int S, int rate, float ceiling,
                    float lookahead_ms, float release_ms, float* y, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  LmParams p;
  int rc = lm_args(ctx, "limit_host", B, S, rate, ceiling, lookahead_ms, release_ms, &p);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("limit_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  if (gain_db)
    for (int b = 0; b < B; ++b)
      if (!(gain_db[b] >= -70.f && gain_db[b] <= 70.f))
        return ctx->fail(VTTS_ERR_BAD_ARG, "limit_host: gain_db[%d]=%g outside [-70, 70]", b, (double)gain_db[b]);
  const size_t o_g = hs.in(gain_db, (size_t)B * 4), o_r = hs.out((size_t)B * 4, reduction_db), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) {
    return lm_launch(ctx, p, rate, hs.x(), hs.n(), gain_db ? hs.dev<const float>(o_g) : nullptr, B, S, hs.dev<float>(o_y), hs.dev<float>(o_r), st);
  });
}

int vtts_loudness_normalize_limited(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float target,
                                    float ceiling, float lookahead_ms, float release_ms, float* y_dev, float* gain_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  LmParams p;
  const int rc = lnl_args(ctx, "loudness_normalize_limited", B, S, rate, target, ceiling, lookahead_ms, release_ms, &p);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "loudness_normalize_limited: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return lnl_launch(ctx, p, x_dev, n_dev, B, S, rate, target, y_dev, gain_db_dev, (cudaStream_t)stream);
}

int vtts_loudness_normalize_limited_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float target,
                                         float ceiling, float lookahead_ms, float release_ms, float* y, float* gain_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  LmParams p;
  int rc = lnl_args(ctx, "loudness_normalize_limited_host", B, S, rate, target, ceiling, lookahead_ms, release_ms, &p);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("loudness_normalize_limited_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_g = hs.out((size_t)B * 4, gain_db), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return lnl_launch(ctx, p, hs.x(), hs.n(), B, S, rate, target, hs.dev<float>(o_y), hs.dev<float>(o_g), st); });
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and samples released in E.
// The window carries H = 2 W + 64 samples: tau of the earliest sample a push needs reads inputs from t - W + 1 - 2 D - 1
// on, t >= P0 - look, that is 2 W + 40 back.
struct vtts_limiter_stream : SampleStream<LmRow, RsRow> {
  using SampleStream::SampleStream;
  int rate = 0, look = 0, pitch = 0;
  LmParams p{};
  LmBufs w{};
  std::vector<float> gain;           // each slot's pre-gain since its BEGIN
};

int vtts_limiter_stream_lookahead(int rate, float lookahead_ms) {
  if (!rate_ok(rate) || !(lookahead_ms >= 1.f && lookahead_ms <= 20.f)) return VTTS_ERR_BAD_ARG;
  const int W = std::max(1, (int)std::rint((double)lookahead_ms * rate / 1000.0));
  // tau[t + W - 1] reads u up to 4(t + W - 1 + D) + 3, whose last input is floor((j + 4 D) / 4) = t + W - 1 + D + 10
  return W - 1 + D + (OS - 1 + OS * D) / OS;
}

int vtts_limiter_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float ceiling, float lookahead_ms,
                               float release_ms, vtts_limiter_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "limiter_stream_create", out, out_pitch != nullptr, max_streams, max_chunk_samples);
  if (rc) return rc;
  LmParams p;
  rc = lm_params(ctx, "limiter_stream_create", rate, ceiling, lookahead_ms, release_ms, &p);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_limiter_stream> ls(new vtts_limiter_stream(ctx, max_streams, max_chunk_samples, 2 * p.W + 64));
  ls->rate = rate;
  ls->p = p;
  ls->look = vtts_limiter_stream_lookahead(rate, lookahead_ms);
  ls->pitch = max_chunk_samples + ls->look;   // END releases at most n_new + look
  ls->gain.assign(max_streams, 0.f);
  const size_t S = max_streams, nb = lm_blocks_max(ls->pitch);
  rc = stream_alloc(ctx, "limiter_stream_create", *ls, [&](Arena& a) {
    ls->carve_window(a);
    ls->w.v = a.take<float>(S * ls->cap);
    ls->w.tau = a.take<float>(S * ls->cap);
    ls->w.alpha = a.take<float>(S * ls->cap);
    ls->w.u = a.take<float>(S * OS * ls->cap);
    ls->w.maps = a.take<float4>(S * nb);
    ls->w.din = a.take<float>(S * nb);
    ls->w.gmin = a.take<float>(S * nb);
    ls->w.start = a.take<float4>(S);
    ls->w.carry_map = a.take<float4>(S);
    ls->w.carry_din = a.take<float>(S);
    ls->w.carry_min = a.take<float>(S);
    ls->carve_tables(a);
  });
  if (rc) return rc;
  const std::vector<float> ones(S, 1.f);   // no reduction yet
  VTTS_CUDA(cudaMemcpy(ls->w.carry_min, ones.data(), S * sizeof(float), cudaMemcpyHostToDevice));
  ls->w.v_ld = ls->cap;
  ls->w.u_ld = (long long)OS * ls->cap;
  ls->w.ld_blk = (int)nb;
  *out_pitch = ls->pitch;
  *out = ls.release();
  return VTTS_OK;
}

int vtts_limiter_stream_destroy(vtts_ctx* ctx, vtts_limiter_stream* ls) { return stream_destroy(ctx, "limiter_stream_destroy", ls); }

int vtts_limiter_stream_push(vtts_ctx* ctx, vtts_limiter_stream* ls, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                             const float* gain_db, float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "limiter_stream_push", ls, x_dev && n_new && flags && gain_db && y_dev && n_out && reduction_db_dev);
  if (rc) return rc;
  const SlotState& sl = ls->slots;
  rc = sl.check(ctx, "limiter_stream_push", ls->F, n_new, flags, [&](int s) -> int {
    if ((flags[s] & 1) && !(gain_db[s] >= -70.f && gain_db[s] <= 70.f))
      return ctx->fail(VTTS_ERR_BAD_ARG, "limiter_stream_push: gain_db[%d]=%g outside [-70, 70]", s, (double)gain_db[s]);
    return VTTS_OK;
  });
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = ls->S;

  // ---- host bookkeeping: before END sample t is released once P > t + look; END releases the rest ----
  LmRow* rows = ls->rows<0>();
  RsRow* rs = ls->rows<1>();
  std::vector<long long> E1(S);
  long long max_u = 0, max_tn = 0, max_rn = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0), R0 = begin ? 0 : sl.E[s];
    const long long R1 = act ? (end ? P1 : std::max(R0, P1 - ls->look)) : R0;
    const float g = begin ? gain_db[s] : ls->gain[s];
    LmRow r{};
    r.x0 = P0 - ls->K;
    r.u0 = std::max(0LL, OS * r.x0);
    r.n = P1;
    r.r0 = R0;
    r.rn = R1 - R0;
    r.ta = std::max(0LL, R0 - ls->p.W + 1);
    r.tn = r.rn > 0 ? std::max(0LL, std::min(P1, R1 + ls->p.W - 1) - r.ta) : 0;
    r.gain_db = g;
    r.begin = begin;
    rows[s] = r;
    const long long nu = act ? OS * (r.x0 + ls->cap) - r.u0 : 0;
    rs[s] = RsRow{r.x0, std::max(0LL, r.x0), P1, r.u0, nu, nu};
    E1[s] = R1;
    n_out[s] = (int32_t)r.rn;
    max_u = std::max(max_u, nu);
    max_tn = std::max(max_tn, r.tn);
    max_rn = std::max(max_rn, r.rn);
  }
  if (max_rn > ls->pitch || max_u > ls->w.u_ld)
    return ctx->fail(VTTS_ERR_CUDA, "limiter_stream_push: %lld outputs / %lld oversampled (internal bound %d / %lld)", max_rn, max_u, ls->pitch,
                     ls->w.u_ld);

  // ---- device: one table copy, window step, gain, then the limiter's seven launches (nine in all) ----
  rc = ls->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  const LmRow* d_rows = ls->d_rows<0>();
  lm_gain_kernel<<<dim3((ls->cap + THREADS - 1) / THREADS, S), THREADS, 0, st>>>(ls->win, ls->cap, ls->cap, nullptr, nullptr, d_rows, ls->cap,
                                                                                  ls->w.v, ls->w.v_ld, nullptr);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  rc = lm_run(ctx, ls->p, ls->rate, ls->cap, nullptr, d_rows, ls->d_rows<1>(), S, max_u, max_tn, max_rn, ls->w, y_dev, ls->pitch, reduction_db_dev, st);
  if (rc) return rc;
  for (int s = 0; s < S; ++s)
    if (flags[s] & 1) ls->gain[s] = gain_db[s];
  ls->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_limiter_stream_push_host(vtts_ctx* ctx, vtts_limiter_stream* ls, const float* x, const int32_t* n_new, const uint8_t* flags,
                                  const float* gain_db, float* y, int32_t* n_out, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "limiter_stream_push_host", ls, x && y && reduction_db);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ls->S * ls->F * 4), o_y = hs.out((size_t)ls->S * ls->pitch * 4, y),
               o_r = hs.out((size_t)ls->S * 4, reduction_db);
  return hs.run([&](cudaStream_t st) {
    return vtts_limiter_stream_push(ctx, ls, hs.dev<const float>(o_x), n_new, flags, gain_db, hs.dev<float>(o_y), n_out, hs.dev<float>(o_r), st);
  });
}
