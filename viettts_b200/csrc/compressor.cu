// Feed-forward compressor of one mono row, fp32 on the device in every vtts_precision mode (oracle/compressor_oracle.py
// states it in float64):
//   L = 20 log10 |x|;  x_L = L - G(L), G the soft-knee gain computer (threshold T, ratio R, knee W; exactly 0 below the
//   knee and at L = -inf);  release y1[t] = max(x_L[t], a_R y1[t - 1] + b_R x_L[t]);  attack
//   y_L[t] = a_A y_L[t - 1] + b_A y1[t] (both from 0);  y = (x m) 10^(-y_L / 20);  reduction = -max y_L.
// a = fp32(exp(-1000 / (tau rate))) and b = 1 - a, exact in fp32 (a >= 0.78 over the parameter ranges), so each stage's
// DC gain b / (1 - a) is 1 to fp32 precision.
//
// Invariant (as in limiter.cu).  Both stages scan as maps over blocks of Q = 256 samples fixed by absolute index.  The
// release steps are the limiter's monotone maps (Map, map_fold, map_apply in vtts_internal.cuh) with a = x_L[t]; the
// attack steps are the affine maps d -> fma(a_A, d, b_A y1[t]), held as Maps with c = -inf (map_apply is then exactly
// the affine map), composing as (m, k) -> (a_A m, fma(a_A, k, b_A y1)).  Per stage: a fold kernel (one thread per
// (row, block)) folds the block's maps in sample order, a chain kernel (one thread per row) walks the block maps from 0
// (or the carried value) to each block's entering value, and the next kernel refolds the block from it.  x_L is
// recomputed from x in every pass.  A row therefore gives the same bits alone, in any batch position, in every
// precision mode, and through the stream at any push pattern.  Rows below the knee (and R = 1) have y_L = 0 everywhere
// and come back as x m bit for bit.
//
// Stream.  No lookahead: every push releases the samples it brings, read where they are (no window).  Per slot the
// partial release and attack maps of the block holding its next sample, that block's y1 and y_L entering values, and
// the running maximum of y_L.  Every push issues the same six launches after its one table copy.
#include <algorithm>
#include <cmath>

#include "stream_common.cuh"

namespace {

constexpr int Q = 256;                // block of both scans
constexpr int SCAN_THREADS = 128;     // one thread per block or row

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

// y[t] = (x[t] m) 10^(-y_L[t] / 20) over call block i of the outputs, both stages refolded from their entering values
// (0 past the compressed samples); bmax[row][i] = the block's largest y_L.  y may be x: every sample is read and
// written by one thread, after the fold kernels have read it.
__global__ void __launch_bounds__(SCAN_THREADS) cp_apply_kernel(const float* x, long long x_ld, int S, const int* __restrict__ n_in,
                                                                const CpRow* __restrict__ rows, const CpParams p,
                                                                const float4* __restrict__ rstart, const float* __restrict__ rdin,
                                                                const float4* __restrict__ astart, const float* __restrict__ adin, int ld_blk,
                                                                float* y, long long y_ld, float* __restrict__ bmax) {
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
  float mx = 0.f;
  for (long long t = lo; t < hi; ++t) {
    if (t >= end) {
      yr[t] = 0.f;
      continue;
    }
    const float v = xr[t];
    map_fold(R, cp_reduction(p, v), p.aR, p.bR);
    cp_attack_fold(A, map_apply(R, y1_in), p.aA, p.bA);
    const float yl = map_apply(A, yl_in);
    const float g = yl > 0.f ? exp10f(-yl / 20.f) : 1.f;
    yr[t] = (v * p.m) * g;
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

int cp_check(vtts_ctx* ctx, const char* who, int B, int S) {
  if (B < 1 || B > 65535 || S < 1 || S > (1 << 30)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: B=%d S=%d (1..65535, 1..2^30)", who, B, S);
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

size_t cp_oneshot_bytes(int B, int S) {
  const size_t nb = cp_blocks_max(S);
  return 2 * al((size_t)B * nb * 16) + 3 * al((size_t)B * nb * 4) + 2 * al((size_t)B * 16);
}

// the six launches of a call: release fold, release chain, attack fold, attack chain, apply, finish
int cp_run(vtts_ctx* ctx, const CpParams& p, const float* x, long long x_ld, int S, const int* n_in, const CpRow* rows, int B,
           long long max_rn, long long max_zn, const CpBufs& w, float* y, long long y_ld, float* red, cudaStream_t st) {
  const dim3 fgrid((unsigned)std::max(1, (cp_blocks_max(max_rn) + SCAN_THREADS - 1) / SCAN_THREADS), B);
  const dim3 agrid((unsigned)std::max(1, (cp_blocks_max(max_zn) + SCAN_THREADS - 1) / SCAN_THREADS), B);
  const unsigned rgrid = (unsigned)((B + SCAN_THREADS - 1) / SCAN_THREADS);
  cp_release_fold_kernel<<<fgrid, SCAN_THREADS, 0, st>>>(x, x_ld, S, n_in, rows, p, w.carry_r, w.rmaps, w.ld_blk, w.rstart);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_chain_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.rmaps, w.ld_blk, w.rdin, w.carry_y1, w.carry_r);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_attack_fold_kernel<<<fgrid, SCAN_THREADS, 0, st>>>(x, x_ld, S, n_in, rows, p, w.rstart, w.rdin, w.carry_a, w.amaps, w.ld_blk, w.astart);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_chain_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.amaps, w.ld_blk, w.adin, w.carry_yl, w.carry_a);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_apply_kernel<<<agrid, SCAN_THREADS, 0, st>>>(x, x_ld, S, n_in, rows, p, w.rstart, w.rdin, w.astart, w.adin, w.ld_blk, y, y_ld, w.bmax);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  cp_finish_kernel<<<rgrid, SCAN_THREADS, 0, st>>>(S, n_in, rows, B, w.bmax, w.ld_blk, w.carry_max, red);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace

int vtts_compress(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float threshold_db, float ratio,
                  float knee_db, float attack_ms, float release_ms, float makeup_db, float* y_dev, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  CpParams p;
  int rc = cp_params(ctx, "compress", rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, &p);
  if (!rc) rc = cp_check(ctx, "compress", B, S);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "compress: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  rc = ctx->ensure_ws(cp_oneshot_bytes(B, S));
  if (rc) return rc;
  CpBufs w{};
  Arena a(ctx->ws, SIZE_MAX, false);
  cp_carve(a, B, cp_blocks_max(S), &w);
  return cp_run(ctx, p, x_dev, S, S, n_dev, nullptr, B, S, S, w, y_dev, S, reduction_db_dev, (cudaStream_t)stream);
}

int vtts_compress_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float threshold_db, float ratio,
                       float knee_db, float attack_ms, float release_ms, float makeup_db, float* y, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  CpParams p;
  int rc = cp_params(ctx, "compress_host", rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, &p);
  if (!rc) rc = cp_check(ctx, "compress_host", B, S);
  if (!rc) rc = host_lengths_check(ctx, "compress_host", n_in, B, S);
  if (rc) return rc;
  if (!x || !y) return ctx->fail(VTTS_ERR_BAD_ARG, "compress_host: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)B * S * 4, r_b = (size_t)B * 4;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, x_b), o_n = hs.in(n_in, r_b), o_r = hs.out(r_b), o_y = hs.out(x_b);
  rc = hs.upload();
  if (!rc)
    rc = vtts_compress(ctx, hs.dev<const float>(o_x), n_in ? hs.dev<const int32_t>(o_n) : nullptr, B, S, rate, threshold_db, ratio, knee_db,
                       attack_ms, release_ms, makeup_db, hs.dev<float>(o_y), hs.dev<float>(o_r), hs.st);
  if (!rc) rc = hs.fetch(o_y, y, x_b);
  if (!rc && reduction_db) rc = hs.fetch(o_r, reduction_db, r_b);
  return rc ? rc : hs.finish();
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and released in E (the same: no lookahead).  A push reads x_dev
// and writes y_dev in place of a window: slot s's new samples [P0, P1) sit at x_dev[s][0, n_new[s]).
struct vtts_compressor_stream : SampleStream<CpRow> {
  using SampleStream::SampleStream;
  CpParams p{};
  CpBufs w{};
};

int vtts_compressor_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float threshold_db, float ratio,
                                  float knee_db, float attack_ms, float release_ms, float makeup_db, vtts_compressor_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!out) return ctx->fail(VTTS_ERR_BAD_ARG, "compressor_stream_create: null output pointer");
  *out = nullptr;
  CpParams p;
  int rc = cp_params(ctx, "compressor_stream_create", rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, &p);
  if (rc) return rc;
  if (max_streams < 1 || max_streams > 65535 || max_chunk_samples < 1 || max_chunk_samples > (1 << 22))
    return ctx->fail(VTTS_ERR_BAD_ARG, "compressor_stream_create: max_streams=%d max_chunk_samples=%d (1..65535, 1..%d)", max_streams,
                     max_chunk_samples, 1 << 22);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_compressor_stream> cs(new vtts_compressor_stream(ctx, max_streams, max_chunk_samples, 0));
  cs->p = p;
  const size_t S = max_streams;
  rc = stream_alloc(ctx, "compressor_stream_create", *cs, [&](Arena& a) {
    cp_carve(a, S, cp_blocks_max(max_chunk_samples), &cs->w);
    cs->w.carry_r = a.take<float4>(S);
    cs->w.carry_a = a.take<float4>(S);
    cs->w.carry_y1 = a.take<float>(S);
    cs->w.carry_yl = a.take<float>(S);
    cs->w.carry_max = a.take<float>(S);
    cs->carve_tables(a);
  });
  if (rc) return rc;
  *out = cs.release();
  return VTTS_OK;
}

int vtts_compressor_stream_destroy(vtts_ctx* ctx, vtts_compressor_stream* cs) { return stream_destroy(ctx, "compressor_stream_destroy", cs); }

int vtts_compressor_stream_push(vtts_ctx* ctx, vtts_compressor_stream* cs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "compressor_stream_push", cs, x_dev && n_new && flags && y_dev && n_out && reduction_db_dev);
  if (rc) return rc;
  const SlotState& sl = cs->slots;
  rc = sl.check(ctx, "compressor_stream_push", cs->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int S = cs->S;

  // ---- host bookkeeping: every sample is released in the push that brings it ----
  CpRow* rows = cs->rows<0>();
  std::vector<long long> E1(S);
  long long max_rn = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    CpRow r{};
    r.x0 = r.r0 = P0;
    r.rn = r.zn = P1 - P0;
    r.begin = begin;
    rows[s] = r;
    E1[s] = P1;
    n_out[s] = (int32_t)(P1 - P0);
    max_rn = std::max(max_rn, r.rn);
  }

  // ---- device: one table copy, then the compressor's six launches ----
  rc = cs->upload_rows(st);
  if (rc) return rc;
  rc = cp_run(ctx, cs->p, x_dev, cs->F, cs->F, nullptr, cs->d_rows<0>(), S, max_rn, max_rn, cs->w, y_dev, cs->F, reduction_db_dev, st);
  if (rc) return rc;
  cs->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_compressor_stream_push_host(vtts_ctx* ctx, vtts_compressor_stream* cs, const float* x, const int32_t* n_new, const uint8_t* flags,
                                     float* y, int32_t* n_out, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "compressor_stream_push_host", cs, x && y && reduction_db);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)cs->S * cs->F * 4, r_b = (size_t)cs->S * 4;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, x_b), o_y = hs.out(x_b), o_r = hs.out(r_b);
  rc = hs.upload();
  if (!rc) rc = vtts_compressor_stream_push(ctx, cs, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, hs.dev<float>(o_r), hs.st);
  if (!rc) rc = hs.fetch(o_y, y, x_b);
  if (!rc) rc = hs.fetch(o_r, reduction_db, r_b);
  return rc ? rc : hs.finish();
}
