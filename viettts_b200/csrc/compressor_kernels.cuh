// The compressor's parameters, scan kernels and launch sequence (compressor.cu states the definition and the block
// invariant), shared by the compressor, the de-esser (deesser.cu), whose detector reads its high band as the level
// source, and the bed ducker (bed.cu), whose gain acts on a second signal.  Internal to each translation unit that
// includes it.
#pragma once
#include <algorithm>
#include <cmath>

#include "stream_common.cuh"

namespace {
namespace cpk {

constexpr int Q = 256;                // block of both scans
constexpr int SCAN_THREADS = 128;     // one thread per block or row
constexpr long long S_MAX = 1 << 30;  // one-shot row length: int sample indices one block past the row stay exact

struct CpRow {
  long long x0;      // absolute index of x buffer element 0
  long long r0;      // absolute index of the call's first sample (y element 0)
  long long rn;      // samples compressed: [r0, r0 + rn)
  long long zn;      // outputs written: [r0, r0 + zn), 0 at or past r0 + rn
  int begin;         // the carried state restarts
  int pad[3];
};
static_assert(sizeof(CpRow) % 16 == 0, "table entries keep 16-byte alignment");

// the fp32 constants of a call, passed by value to every kernel
struct CpParams {
  float T;           // threshold dBFS
  float hw;          // W / 2
  float s;           // 1 - 1 / R, the slope of x_L above the knee
  float q;           // (1 - 1 / R) / (2 W) inside the knee (0 for the hard knee)
  float aR, bR;      // release
  float aA, bA;      // attack
  float m;           // makeup factor
};

// rows == nullptr: the one-shot row b, n = n_in[b] clamped to [0, S], outputs [0, S)
__device__ __forceinline__ CpRow cp_row(const CpRow* rows, const int* n_in, int S, int b) {
  if (rows) return rows[b];
  CpRow r;
  r.x0 = r.r0 = 0;
  r.rn = n_in ? min(max(n_in[b], 0), S) : S;
  r.zn = S;
  r.begin = 1;
  return r;
}

// call blocks over the n samples from r0
__device__ __forceinline__ int cp_blocks(long long r0, long long n) { return n > 0 ? (int)((r0 + n - 1) / Q - r0 / Q + 1) : 0; }

// the samples [lo, hi) of call block i over the n samples from r0
__device__ __forceinline__ void cp_block_span(long long r0, long long n, int i, long long& lo, long long& hi) {
  const long long kb = r0 / Q + i;
  lo = max(r0, kb * Q);
  hi = min(r0 + n, (kb + 1) * Q);
}

__device__ __forceinline__ Map cp_map(const float4& v) { return Map{v.x, v.y, v.z}; }
__device__ __forceinline__ float4 cp_f4(const Map& M) { return make_float4(M.c, M.m, M.k, 0.f); }

// x_L of one sample: the gain computer's reduction in dB (>= 0)
__device__ __forceinline__ float cp_reduction(const CpParams& p, float x) {
  const float over = 20.f * log10f(fabsf(x)) - p.T;
  if (!(over >= -p.hw)) return 0.f;      // below the knee, and L = -inf
  if (over > p.hw) return p.s * over;
  const float u = over + p.hw;
  return p.q * u * u;
}

// the attack step d -> fma(a, d, b y1) after M
__device__ __forceinline__ void cp_attack_fold(Map& M, float y1, float a, float b) {
  M.m = a * M.m;
  M.k = fmaf(a, M.k, b * y1);
}

// maps[row][i] = the release fold of call block i, from the carried partial map for i = 0 (stream rows that do not
// begin), else from the identity; start[row] = block 0's starting map
__global__ void __launch_bounds__(SCAN_THREADS) cp_release_fold_kernel(const float* x, long long x_ld, int S, const int* __restrict__ n_in,
                                                                       const CpRow* __restrict__ rows, const CpParams p,
                                                                       const float4* __restrict__ carry, float4* __restrict__ maps, int ld_blk,
                                                                       float4* __restrict__ start) {
  const int b = blockIdx.y, i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  const CpRow r = cp_row(rows, n_in, S, b);
  if (i >= cp_blocks(r.r0, r.rn)) return;
  Map M = map_id();
  if (i == 0) {
    if (carry && !r.begin) M = cp_map(carry[b]);
    start[b] = cp_f4(M);
  }
  long long lo, hi;
  cp_block_span(r.r0, r.rn, i, lo, hi);
  const float* xr = x + (size_t)b * x_ld - r.x0;
  for (long long t = lo; t < hi; ++t) map_fold(M, cp_reduction(p, xr[t]), p.aR, p.bR);
  maps[(size_t)b * ld_blk + i] = cp_f4(M);
}

// din[row][i] = the value entering call block i: d <- M_i(d) over the call blocks that end at a block boundary, from
// the carried value (0 when the row begins); the carry takes the entering value and the partial map of the block
// holding the row's next sample.  Runs once per stage.
__global__ void __launch_bounds__(SCAN_THREADS) cp_chain_kernel(int S, const int* __restrict__ n_in, const CpRow* __restrict__ rows, int B,
                                                                const float4* __restrict__ maps, int ld_blk, float* __restrict__ din,
                                                                float* carry_din, float4* carry_map) {
  const int b = blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (b >= B) return;
  const CpRow r = cp_row(rows, n_in, S, b);
  const int nb = cp_blocks(r.r0, r.rn);
  float d = (carry_din && !r.begin) ? carry_din[b] : 0.f;
  float4 part = cp_f4(map_id());
  if (carry_map && !r.begin) part = carry_map[b];
  for (int i = 0; i < nb; ++i) {
    din[(size_t)b * ld_blk + i] = d;
    long long lo, hi;
    cp_block_span(r.r0, r.rn, i, lo, hi);
    const float4 M = maps[(size_t)b * ld_blk + i];
    if (hi % Q == 0) {
      d = map_apply(cp_map(M), d);
      part = cp_f4(map_id());
    } else {
      part = M;
    }
  }
  if (carry_din) {
    carry_din[b] = d;
    carry_map[b] = part;
  }
}

// amaps[row][i] = the attack fold of call block i over y1[t] = (release fold up to t)(y1 entering), the release refolded
// from rstart (block 0) or the identity; the attack from the carried partial map for block 0 (stream rows that do not
// begin), else the identity; astart[row] = block 0's starting attack map
__global__ void __launch_bounds__(SCAN_THREADS) cp_attack_fold_kernel(const float* x, long long x_ld, int S, const int* __restrict__ n_in,
                                                                      const CpRow* __restrict__ rows, const CpParams p,
                                                                      const float4* __restrict__ rstart, const float* __restrict__ rdin,
                                                                      const float4* __restrict__ carry, float4* __restrict__ amaps, int ld_blk,
                                                                      float4* __restrict__ astart) {
  const int b = blockIdx.y, i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  const CpRow r = cp_row(rows, n_in, S, b);
  if (i >= cp_blocks(r.r0, r.rn)) return;
  Map R = map_id(), A = map_id();
  if (i == 0) {
    R = cp_map(rstart[b]);
    if (carry && !r.begin) A = cp_map(carry[b]);
    astart[b] = cp_f4(A);
  }
  const float y1_in = rdin[(size_t)b * ld_blk + i];
  long long lo, hi;
  cp_block_span(r.r0, r.rn, i, lo, hi);
  const float* xr = x + (size_t)b * x_ld - r.x0;
  for (long long t = lo; t < hi; ++t) {
    map_fold(R, cp_reduction(p, xr[t]), p.aR, p.bR);
    cp_attack_fold(A, map_apply(R, y1_in), p.aA, p.bA);
  }
  amaps[(size_t)b * ld_blk + i] = cp_f4(A);
}

// The output rule of the apply kernel, a template parameter so that each user compiles only its own: where the
// detector reads its level (the fold kernels read the same source), the cap on y_L of row b, and y of row b at absolute
// sample t from the sample x, its level sample l and g = 10^(-y_L / 20) (1 exactly where the capped y_L is 0).  The
// compressor and the de-esser ignore the row and the sample index.
struct CpMakeup {                   // the compressor: level source x, y = (x m) g
  __host__ __device__ const float* source(const float* x) const { return x; }
  __device__ __forceinline__ float level(const float* xr, long long t, float v) const { return v; }
  __device__ __forceinline__ float cap(int, float yl) const { return yl; }
  __device__ __forceinline__ float out(const CpParams& p, int, long long, float v, float l, float yl, float g) const { return (v * p.m) * g; }
};

struct CpSplit {                    // the de-esser: level source its high band h (x's layout), y = x - (1 - g) h
  const float* h;
  float range;                      // the cap on y_L, dB
  __host__ __device__ const float* source(const float*) const { return h; }
  __device__ __forceinline__ float level(const float* xr, long long t, float) const { return xr[t]; }
  __device__ __forceinline__ float cap(int, float yl) const { return fminf(yl, range); }
  __device__ __forceinline__ float out(const CpParams&, int, long long, float v, float l, float yl, float g) const {
    return yl > 0.f ? fmaf(g - 1.f, l, v) : v;
  }
};

// y[t] = out(x[t], l[t], g[t]) over call block i of the outputs, both stages refolded from their entering values (0
// past the compressed samples); bmax[row][i] = the block's largest capped y_L.  y may be x: every sample is read and
// written by one thread, after the fold kernels have read it.
template <class Out>
__global__ void __launch_bounds__(SCAN_THREADS) cp_apply_kernel(const float* x, long long x_ld, int S, const int* __restrict__ n_in,
                                                                const CpRow* __restrict__ rows, const CpParams p,
                                                                const float4* __restrict__ rstart, const float* __restrict__ rdin,
                                                                const float4* __restrict__ astart, const float* __restrict__ adin, int ld_blk,
                                                                float* y, long long y_ld, float* __restrict__ bmax, const Out o) {
  const int b = blockIdx.y, i = blockIdx.x * SCAN_THREADS + threadIdx.x;
  const CpRow r = cp_row(rows, n_in, S, b);
  if (i >= cp_blocks(r.r0, r.zn)) return;
  long long lo, hi;
  cp_block_span(r.r0, r.zn, i, lo, hi);
  float* yr = y + (size_t)b * y_ld - r.r0;
  const long long end = r.r0 + r.rn;
  if (lo >= end) {                       // one-shot blocks past the row's end
    for (long long t = lo; t < hi; ++t) yr[t] = 0.f;
    return;
  }
  Map R = map_id(), A = map_id();
  if (i == 0) {
    R = cp_map(rstart[b]);
    A = cp_map(astart[b]);
  }
  const float y1_in = rdin[(size_t)b * ld_blk + i], yl_in = adin[(size_t)b * ld_blk + i];
  const float* xr = x + (size_t)b * x_ld - r.x0;
  const float* lr = o.source(x) + (size_t)b * x_ld - r.x0;
  float mx = 0.f;
  for (long long t = lo; t < hi; ++t) {
    if (t >= end) {
      yr[t] = 0.f;
      continue;
    }
    const float v = xr[t], l = o.level(lr, t, v);
    map_fold(R, cp_reduction(p, l), p.aR, p.bR);
    cp_attack_fold(A, map_apply(R, y1_in), p.aA, p.bA);
    const float yl = o.cap(b, map_apply(A, yl_in));
    const float g = yl > 0.f ? exp10f(-yl / 20.f) : 1.f;
    yr[t] = o.out(p, b, t, v, l, yl, g);
    mx = fmaxf(mx, yl);
  }
  bmax[(size_t)b * ld_blk + i] = mx;
}

// red[row] = -(the largest y_L over the call's blocks and the carried maximum of stream rows that do not begin)
__global__ void __launch_bounds__(SCAN_THREADS) cp_finish_kernel(int S, const int* __restrict__ n_in, const CpRow* __restrict__ rows, int B,
                                                                 const float* __restrict__ bmax, int ld_blk, float* carry_max,
                                                                 float* __restrict__ red) {
  const int b = blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (b >= B) return;
  const CpRow r = cp_row(rows, n_in, S, b);
  float g = (carry_max && !r.begin) ? carry_max[b] : 0.f;
  const int nb = cp_blocks(r.r0, r.rn);
  for (int i = 0; i < nb; ++i) g = fmaxf(g, bmax[(size_t)b * ld_blk + i]);
  if (carry_max) carry_max[b] = g;
  if (red) red[b] = 0.f - g;
}

int cp_params(vtts_ctx* ctx, const char* who, int rate, float threshold_db, float ratio, float knee_db, float attack_ms, float release_ms,
              float makeup_db, CpParams* p) {
  if (rate < 8000 || rate > 192000) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rate %d (in [8000, 192000])", who, rate);
  if (!(threshold_db >= -60.f && threshold_db <= 0.f))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: threshold %g dBFS (in [-60, 0])", who, (double)threshold_db);
  if (!(ratio >= 1.f && ratio <= 20.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: ratio %g (in [1, 20])", who, (double)ratio);
  if (!(knee_db >= 0.f && knee_db <= 24.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: knee %g dB (in [0, 24])", who, (double)knee_db);
  if (!(attack_ms >= 0.5f && attack_ms <= 200.f))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: attack %g ms (in [0.5, 200])", who, (double)attack_ms);
  if (!(release_ms >= 5.f && release_ms <= 5000.f))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: release %g ms (in [5, 5000])", who, (double)release_ms);
  if (!(makeup_db >= -24.f && makeup_db <= 24.f))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: makeup %g dB (in [-24, 24])", who, (double)makeup_db);
  const double s = 1.0 - 1.0 / (double)ratio;
  p->T = threshold_db;
  p->hw = 0.5f * knee_db;
  p->s = (float)s;
  p->q = knee_db > 0.f ? (float)(s / (2.0 * (double)knee_db)) : 0.f;
  p->aR = (float)std::exp(-1000.0 / ((double)release_ms * rate));
  p->bR = 1.f - p->aR;
  p->aA = (float)std::exp(-1000.0 / ((double)attack_ms * rate));
  p->bA = 1.f - p->aA;
  p->m = (float)std::pow(10.0, (double)makeup_db / 20.0);
  return VTTS_OK;
}

size_t al(size_t b) { return (b + 255) & ~size_t(255); }

int cp_blocks_max(long long n) { return (int)(n / Q + 2); }

// the buffers of one call: per call block the two stages' maps and entering values and the largest y_L, per row the
// two starting maps; a stream adds its carries
struct CpBufs {
  float4 *rmaps, *amaps, *rstart, *astart;
  float *rdin, *adin, *bmax;
  int ld_blk;
  float4 *carry_r, *carry_a;          // stream: [rows] carried partial maps, else null
  float *carry_y1, *carry_yl;         // stream: [rows] carried entering values, else null
  float* carry_max;                   // stream: [rows] running largest y_L, else null
};

void cp_carve(Arena& a, size_t rows, int nb, CpBufs* w) {
  w->rmaps = a.take<float4>(rows * nb);
  w->amaps = a.take<float4>(rows * nb);
  w->rdin = a.take<float>(rows * nb);
  w->adin = a.take<float>(rows * nb);
  w->bmax = a.take<float>(rows * nb);
  w->rstart = a.take<float4>(rows);
  w->astart = a.take<float4>(rows);
  w->ld_blk = nb;
}

// the stream row of a slot that holds P0 samples before the push and P1 after it: the push's inputs are read where they
// are, and every sample it brings is released
CpRow cp_stream_row(long long P0, long long P1, int begin) {
  CpRow r{};
  r.x0 = r.r0 = P0;
  r.rn = r.zn = P1 - P0;
  r.begin = begin;
  return r;
}

size_t cp_oneshot_bytes(int B, int S) {
  const size_t nb = cp_blocks_max(S);
  return 2 * al((size_t)B * nb * 16) + 3 * al((size_t)B * nb * 4) + 2 * al((size_t)B * 16);
}

// the six launches of a call: release fold, release chain, attack fold, attack chain, apply, finish; the fold kernels
// read their level from o.source(x)
template <class Out = CpMakeup>
int cp_run(vtts_ctx* ctx, const CpParams& p, const float* x, long long x_ld, int S, const int* n_in, const CpRow* rows, int B,
           long long max_rn, long long max_zn, const CpBufs& w, float* y, long long y_ld, float* red, cudaStream_t st, const Out& o = Out{}) {
  const dim3 fgrid((unsigned)std::max(1, (cp_blocks_max(max_rn) + SCAN_THREADS - 1) / SCAN_THREADS), B);
  const dim3 agrid((unsigned)std::max(1, (cp_blocks_max(max_zn) + SCAN_THREADS - 1) / SCAN_THREADS), B);
  const unsigned rgrid = (unsigned)((B + SCAN_THREADS - 1) / SCAN_THREADS);
  cp_release_fold_kernel<<<fgrid, SCAN_THREADS, 0, st>>>(o.source(x), x_ld, S, n_in, rows, p, w.carry_r, w.rmaps, w.ld_blk, w.rstart);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_chain_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.rmaps, w.ld_blk, w.rdin, w.carry_y1, w.carry_r);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_attack_fold_kernel<<<fgrid, SCAN_THREADS, 0, st>>>(o.source(x), x_ld, S, n_in, rows, p, w.rstart, w.rdin, w.carry_a, w.amaps, w.ld_blk, w.astart);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_chain_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.amaps, w.ld_blk, w.adin, w.carry_yl, w.carry_a);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_apply_kernel<<<agrid, SCAN_THREADS, 0, st>>>(x, x_ld, S, n_in, rows, p, w.rstart, w.rdin, w.astart, w.adin, w.ld_blk, y, y_ld, w.bmax,
                                                  o);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_finish_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.bmax, w.ld_blk, w.carry_max, red);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace cpk
}  // namespace
