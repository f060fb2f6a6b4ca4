// Loudness meter and normalizer (ITU-R BS.1770-4 gated loudness of one mono row, plus a true peak), fp32 on the device
// in every vtts_precision mode.
//   K-weighting: the libebur128 shelf and high-pass biquads for the row's rate, designed in double, rounded to fp32
//   once and cached in the context per rate; state s = (z1, z2, s1, s2) from zero at sample 0.  The shelf runs in
//   transposed direct form II.  The high-pass runs as the trapezoidal (TPT) state-variable filter of the same bilinear
//   transform, whose coefficients are g = tan(pi f0 / r) and 1 / Q instead of a1 = -2 + O(g) and a2 = 1 - O(g): rounded
//   to fp32, direct-form coefficients move the 38 Hz poles by up to 0.5 % at 48 kHz, which a 50 Hz tone reads as
//   1e-3 LU; the state-variable form keeps the poles to fp32 precision.
//   Sub-blocks of m = rate / 10 samples: E_k = sum of y^2; blocks j < J = max(0, K - 3) of four sub-blocks, K = floor(n / m);
//   z_j = (E_j + .. + E_j+3) / 4m, l_j = -0.691 + 10 log10 z_j; absolute gate -70, relative gate -10 LU; momentary l_J-1;
//   short-term over the last 30 sub-blocks; true peak max(|x|, |resample_poly(x, 4, 1)|) in dBTP.
//
// Energy invariant.  E_k and e_k (the sub-block's end state from zero) are fixed fp32 functions of the state s_k entering
// sub-block k and of its m samples; the state chain is s_k+1 = M s_k + e_k with M = A^m (A the 4 x 4 state matrix of the
// cascade, powered in double and rounded to fp32).  Every reduction has an order fixed by the sub-block or block index,
// so a row gives the same bits alone, in any batch, and through the stream.
//
// Sub-block kernel.  One warp per (row, sub-block).  Lane l filters samples [l seg, (l + 1) seg) (seg = ceil(m / 32))
// from zero state (lane 0 from s_k in the energy pass); a Hillis-Steele scan with the segment transitions A^(seg d)
// composes the lane end states into each lane's entering state; each lane re-filters its segment from that state, summing
// y^2 in sample order, and a fixed shuffle tree gives E_k.  Lanes past the last sample hold no samples, and every lane
// before it holds exactly seg, so the scan's constant transitions are the right ones wherever they are used.  The kernel
// runs twice: from zero (e_k, written by the lane holding the sub-block's last sample) and from s_k (E_k).
//
// Chain kernel.  One thread per row walks s_k+1 = M s_k + e_k over the row's sub-blocks (36 000 steps for an hour at any
// rate).  Gate kernel.  One CTA per row: z_j, both gates, the readings, the peak from the per-tile maxima and the gain.
//
// Stream.  Per slot a window of m carried samples plus one chunk (the resample stream's window step), the state at the
// last complete sub-block boundary, the E_k history and the running peak; every push issues the same seven launches.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "stream_common.cuh"

namespace {

using LnFilter = vtts_ctx::LnFilter;

constexpr int LN_WARPS = 4;           // sub-blocks per CTA
constexpr int CHAIN_THREADS = 128;
constexpr int GATE_THREADS = 256;
constexpr int PEAK_THREADS = 256;
constexpr int PEAK_TILE = PEAK_THREADS * 16;
constexpr int APPLY_THREADS = 256;
constexpr int OS = 4;                 // true-peak oversampling (resample_poly(x, 4, 1))
constexpr unsigned FULL = 0xffffffffu;

struct LnRow {
  long long x0;      // absolute sample index of buffer element 0
  long long k0;      // first sub-block processed
  long long nu;      // oversampled outputs scanned for the peak (u elements [0, nu))
  int nk;            // sub-blocks processed
  int K;             // complete sub-blocks of the row (the gate's extent)
  int xa, nx;        // samples scanned for the peak: buffer elements [xa, xa + nx)
  int begin;         // the carried state and peak restart
};

// rows == nullptr: the one-shot row b, n = n_in[b] clamped to [0, S] (or S)
__device__ __forceinline__ LnRow ln_row(const LnRow* rows, const int* n_in, int S, int m, int b) {
  if (rows) return rows[b];
  const int n = n_in ? min(max(n_in[b], 0), S) : S;
  LnRow r;
  r.x0 = 0;
  r.k0 = 0;
  r.nk = r.K = n / m;
  r.xa = 0;
  r.nx = n;
  r.nu = (long long)OS * n;
  r.begin = 1;
  return r;
}

// one sample through the cascade: shelf (c[0..4] = b0 b1 b2 a1 a2) then high-pass (c[5..8] = g, g + 1 / Q,
// 1 / (1 + g (g + 1 / Q)), a0, see ln_filter); returns y
__device__ __forceinline__ float kw_step(const float* __restrict__ c, float (&s)[4], float x) {
  const float y1 = fmaf(c[0], x, s[0]);
  s[0] = fmaf(c[1], x, fmaf(-c[3], y1, s[1]));
  s[1] = fmaf(c[2], x, -c[4] * y1);
  const float hp = (y1 - fmaf(c[6], s[2], s[3])) * c[7];
  const float v1 = c[5] * hp;
  const float bp = v1 + s[2];
  s[2] = bp + v1;
  const float v2 = c[5] * bp;
  s[3] = (v2 + s[3]) + v2;
  return c[8] * hp;
}

// r = add + M v (row-major M), fixed order
__device__ __forceinline__ void mat_fma(const float* __restrict__ M, const float (&v)[4], const float (&add)[4], float (&r)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float a = add[i];
#pragma unroll
    for (int j = 0; j < 4; ++j) a = fmaf(M[i * 4 + j], v[j], a);
    r[i] = a;
  }
}

// ENERGY = false: e_out[row][q][4] = the sub-block's end state from zero.  ENERGY = true: lane 0 enters with
// s_in[row][q][4] and E_out[row][k] = sum of y^2 (k absolute).  q = k - k0 indexes the call's sub-blocks.
template <bool ENERGY>
__global__ void __launch_bounds__(LN_WARPS * 32) kw_subblock_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                    const int* __restrict__ n_in, const LnRow* __restrict__ rows,
                                                                    const LnFilter f, int m, int seg, int ld_k,
                                                                    const float* __restrict__ s_in, float* __restrict__ e_out,
                                                                    float* __restrict__ E_out, long long E_ld) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
  const int q = blockIdx.x * LN_WARPS + warp;
  const LnRow r = ln_row(rows, n_in, S, f.rate / 10, b);
  if (q >= r.nk) return;                                  // whole warps leave: only warp shuffles below
  const long long k = r.k0 + q;
  const float* xs = x + (size_t)b * x_ld + (k * m - r.x0);
  const int i0 = min(lane * seg, m), i1 = min(i0 + seg, m);
  float enter[4] = {0.f, 0.f, 0.f, 0.f};
  if (ENERGY && lane == 0) {
    const float4 v = *reinterpret_cast<const float4*>(s_in + ((size_t)b * ld_k + q) * 4);
    enter[0] = v.x; enter[1] = v.y; enter[2] = v.z; enter[3] = v.w;
  }
  float st[4] = {enter[0], enter[1], enter[2], enter[3]};
  for (int i = i0; i < i1; ++i) kw_step(f.coef, st, __ldg(xs + i));
  // inclusive scan of v_l = A^seg v_l-1 + st_l
#pragma unroll
  for (int d = 0; d < 5; ++d) {
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = __shfl_up_sync(FULL, st[j], 1 << d);
    if (lane >= (1 << d)) mat_fma(f.seg[d], o, st, st);
  }
  float s[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float v = __shfl_up_sync(FULL, st[j], 1);
    s[j] = lane == 0 ? enter[j] : v;
  }
  float acc = 0.f;
  for (int i = i0; i < i1; ++i) {
    const float y = kw_step(f.coef, s, __ldg(xs + i));
    if (ENERGY) acc = fmaf(y, y, acc);
  }
  if (ENERGY) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(FULL, acc, o);
    if (lane == 0) E_out[(size_t)b * E_ld + k] = acc;
  } else if (i0 < i1 && i1 == m) {
    *reinterpret_cast<float4*>(e_out + ((size_t)b * ld_k + q) * 4) = make_float4(s[0], s[1], s[2], s[3]);
  }
}

// s_out[row][q] = the state entering sub-block k0 + q: s = M s + e over the row's sub-blocks, from carry[row] (unless the
// row begins) or zero; the final state goes back to carry
__global__ void __launch_bounds__(CHAIN_THREADS) kw_chain_kernel(const int* __restrict__ n_in, const LnRow* __restrict__ rows, int S,
                                                                 int B, const LnFilter f, int ld_k, const float* __restrict__ e,
                                                                 float* __restrict__ s_out, float* __restrict__ carry) {
  const int b = blockIdx.x * CHAIN_THREADS + threadIdx.x;
  if (b >= B) return;
  const LnRow r = ln_row(rows, n_in, S, f.rate / 10, b);
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (carry && !r.begin)
    for (int j = 0; j < 4; ++j) s[j] = carry[b * 4 + j];
  const float4* er = reinterpret_cast<const float4*>(e) + (size_t)b * ld_k;
  float4* so = reinterpret_cast<float4*>(s_out) + (size_t)b * ld_k;
  for (int q = 0; q < r.nk; ++q) {
    so[q] = make_float4(s[0], s[1], s[2], s[3]);
    const float4 v = er[q];
    const float add[4] = {v.x, v.y, v.z, v.w};
    mat_fma(f.blk, s, add, s);
  }
  if (carry)
    for (int j = 0; j < 4; ++j) carry[b * 4 + j] = s[j];
}

__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_down_sync(FULL, v, o));
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_down_sync(FULL, v, o));
  }
  return v;
}

// part[row][t] = max |v| over tile t of the row's peak range: x elements [xa, xa + nx) followed by u elements [0, nu)
__global__ void __launch_bounds__(PEAK_THREADS) peak_kernel(const float* __restrict__ x, long long x_ld, const float* __restrict__ u,
                                                            long long u_ld, int S, const int* __restrict__ n_in,
                                                            const LnRow* __restrict__ rows, int m, float* __restrict__ part, int part_ld) {
  __shared__ float red[PEAK_THREADS / 32];
  const int b = blockIdx.y;
  const LnRow r = ln_row(rows, n_in, S, m, b);
  const long long total = r.nx + r.nu, t0 = (long long)blockIdx.x * PEAK_TILE;
  if (t0 >= total) return;
  const float* xr = x + (size_t)b * x_ld + r.xa;
  const float* ur = u + (size_t)b * u_ld - r.nx;
  const long long t1 = min(total, t0 + PEAK_TILE);
  float v = 0.f;
  for (long long i = t0 + threadIdx.x; i < t1; i += PEAK_THREADS) v = fmaxf(v, fabsf(i < r.nx ? __ldg(xr + i) : __ldg(ur + i)));
  v = block_max(v, red);
  if (threadIdx.x == 0) part[(size_t)b * part_ld + blockIdx.x] = v;
}

// deterministic CTA sum (thread partials in a fixed tree); every thread gets the result
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(FULL, v, o);
  __syncthreads();                                        // red may still be read by a previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < GATE_THREADS / 32 ? red[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(FULL, v, o);
    if (lane == 0) red[GATE_THREADS / 32] = v;
  }
  __syncthreads();
  return red[GATE_THREADS / 32];
}

__device__ __forceinline__ float lufs(float z) { return -0.691f + 10.f * log10f(z); }

// out[row] = (integrated, momentary, short-term, true peak); with gain_f: the normalization gain g (dB) and
// f = fp32(10^(g / 20)) of target / ceiling (ceiling +inf: none)
__global__ void __launch_bounds__(GATE_THREADS) loudness_gate_kernel(const float* __restrict__ E, long long E_ld, int S,
                                                                     const int* __restrict__ n_in, const LnRow* __restrict__ rows,
                                                                     int m, const float* __restrict__ part, int part_ld,
                                                                     float* __restrict__ peak_carry, float* __restrict__ out,
                                                                     float target, float ceiling, float* __restrict__ gain_db,
                                                                     float* __restrict__ gain_f) {
  __shared__ float red[GATE_THREADS / 32 + 1];
  const int b = blockIdx.x, tid = threadIdx.x;
  const LnRow r = ln_row(rows, n_in, S, m, b);
  const float* Er = E + (size_t)b * E_ld;
  const int J = max(0, r.K - 3);
  const float inv4m = 1.f / (float)(4 * m);
  float sa = 0.f, ca = 0.f;
  for (int j = tid; j < J; j += GATE_THREADS) {
    const float z = (((Er[j] + Er[j + 1]) + Er[j + 2]) + Er[j + 3]) * inv4m;
    if (lufs(z) > -70.f) { sa += z; ca += 1.f; }
  }
  sa = block_sum(sa, red);
  ca = block_sum(ca, red);
  const float gamma = ca > 0.f ? lufs(sa / ca) - 10.f : INFINITY;
  float sr = 0.f, cr = 0.f;
  for (int j = tid; j < J; j += GATE_THREADS) {
    const float z = (((Er[j] + Er[j + 1]) + Er[j + 2]) + Er[j + 3]) * inv4m;
    const float l = lufs(z);
    if (l > -70.f && l > gamma) { sr += z; cr += 1.f; }
  }
  sr = block_sum(sr, red);
  cr = block_sum(cr, red);
  const int ntile = (int)((r.nx + r.nu + PEAK_TILE - 1) / PEAK_TILE);
  float p = 0.f;
  for (int t = tid; t < ntile; t += GATE_THREADS) p = fmaxf(p, part[(size_t)b * part_ld + t]);
  __syncthreads();
  p = block_max(p, red);
  if (tid != 0) return;
  if (peak_carry) {
    if (!r.begin) p = fmaxf(p, peak_carry[b]);
    peak_carry[b] = p;
  }
  const float L = cr > 0.f ? lufs(sr / cr) : -INFINITY;
  const float mom = J > 0 ? lufs((((Er[J - 1] + Er[J]) + Er[J + 1]) + Er[J + 2]) * inv4m) : -INFINITY;
  float st = -INFINITY;
  if (r.K >= 30) {
    float e = 0.f;
    for (int k = r.K - 30; k < r.K; ++k) e += Er[k];
    st = lufs(e / (float)(30 * m));
  }
  const float tp = 20.f * log10f(p);
  float* o = out + (size_t)b * 4;
  o[0] = L;
  o[1] = mom;
  o[2] = st;
  o[3] = tp;
  if (gain_f) {
    float g = 0.f;
    if (isfinite(L)) {
      g = target - L;
      if (isfinite(ceiling)) g = fminf(g, ceiling - tp);
    }
    gain_db[b] = g;
    gain_f[b] = (float)exp10((double)g / 20.0);
  }
}

// y = x f[row] for t < n, 0 past it (y may be x)
__global__ void __launch_bounds__(APPLY_THREADS) gain_apply_kernel(const float* x, int S, const int* __restrict__ n_in,
                                                                   const float* __restrict__ f, float* y) {
  const int b = blockIdx.y;
  const long long t = (long long)blockIdx.x * APPLY_THREADS + threadIdx.x;
  if (t >= S) return;
  const int n = n_in ? min(max(n_in[b], 0), S) : S;
  const size_t i = (size_t)b * S + t;
  y[i] = t < n ? x[i] * f[b] : 0.f;
}

bool rate_ok(int rate) { return rate >= 8000 && rate <= 192000 && rate % 10 == 0; }

// shelf then high-pass: b0 b1 b2 a1 a2 each, in double
void ln_design(int rate, double* c) {
  const double pi = 3.14159265358979323846;
  {
    const double f0 = 1681.974450955533, G = 3.999843853973347, Q = 0.7071752369554196;
    const double K = std::tan(pi * f0 / rate), Vh = std::pow(10.0, G / 20.0), Vb = std::pow(Vh, 0.4996667741545416);
    const double a0 = 1.0 + K / Q + K * K;
    c[0] = (Vh + Vb * K / Q + K * K) / a0;
    c[1] = 2.0 * (K * K - Vh) / a0;
    c[2] = (Vh - Vb * K / Q + K * K) / a0;
    c[3] = 2.0 * (K * K - 1.0) / a0;
    c[4] = (1.0 - K / Q + K * K) / a0;
  }
  {
    const double f0 = 38.13547087613982, Q = 0.5003270373253953;
    const double K = std::tan(pi * f0 / rate), a0 = 1.0 + K / Q + K * K;
    c[5] = 1.0;
    c[6] = -2.0;
    c[7] = 1.0;
    c[8] = 2.0 * (K * K - 1.0) / a0;
    c[9] = (1.0 - K / Q + K * K) / a0;
  }
}

int seg_of(int m) { return (m + 31) / 32; }

// the context's fp32 cascade of `rate` (designed at the first use).  The high-pass b = [1, -2, 1] / a equals a0 times
// the bilinear transform of s^2 / (s^2 + s / Q + 1) with K = tan(pi f0 / r), the TPT state-variable filter's high-pass
// output with g = K.
const LnFilter& ln_filter(vtts_ctx* ctx, int rate) {
  for (const auto& f : ctx->ln_filters)
    if (f.rate == rate) return f;
  double c[10];
  ln_design(rate, c);
  const double g = std::tan(3.14159265358979323846 * 38.13547087613982 / rate), kq = 1.0 / 0.5003270373253953;
  const double p[9] = {c[0], c[1], c[2], c[3], c[4], g, g + kq, 1.0 / (1.0 + g * (g + kq)), 1.0 + g * kq + g * g};
  // zero-input state matrix of kw_step: column j = the state after one step from unit state e_j
  double A[16];
  for (int j = 0; j < 4; ++j) {
    double s[4] = {0, 0, 0, 0};
    s[j] = 1.0;
    const double y1 = s[0];
    const double z1 = -p[3] * y1 + s[1], z2 = -p[4] * y1;
    const double hp = (y1 - p[6] * s[2] - s[3]) * p[7];
    const double bp = p[5] * hp + s[2];
    const double col[4] = {z1, z2, bp + p[5] * hp, p[5] * bp + s[3] + p[5] * bp};
    for (int i = 0; i < 4; ++i) A[i * 4 + j] = col[i];
  }
  LnFilter f{};
  f.rate = rate;
  for (int i = 0; i < 9; ++i) f.coef[i] = (float)p[i];
  const int m = rate / 10, seg = seg_of(m);
  double P[16];
  for (int d = 0; d < 5; ++d) {
    vtts_mat_pow(A, (long long)seg << d, P, 4);
    for (int i = 0; i < 16; ++i) f.seg[d][i] = (float)P[i];
  }
  vtts_mat_pow(A, m, P, 4);
  for (int i = 0; i < 16; ++i) f.blk[i] = (float)P[i];
  ctx->ln_filters.push_back(f);
  return ctx->ln_filters.back();
}

// where the stages of one call find their buffers
struct LnBufs {
  float *e, *s, *E, *u, *part;
  int ld_k;              // sub-blocks per row of e / s
  long long E_ld, u_ld;
  int part_ld;
  float* carry;          // stream: [rows][4] filter state, else null
  float* peak;           // stream: [rows] running peak, else null
};

// the six measuring launches: two sub-block passes around the chain, the 4x oversampler, the tile maxima, the gate
int ln_measure(vtts_ctx* ctx, const LnFilter& f, const float* x, long long x_ld, int S, const int* n_in, const LnRow* rows,
               const RsRow* rs_rows, int B, long long max_k, long long max_u, long long max_peak, const LnBufs& w, float* out,
               float target, float ceiling, float* gain_db, float* gain_f, cudaStream_t st) {
  const int m = f.rate / 10, seg = seg_of(m);
  const dim3 sgrid((unsigned)std::max(1LL, (max_k + LN_WARPS - 1) / LN_WARPS), B);
  kw_subblock_kernel<false><<<sgrid, LN_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, f, m, seg, w.ld_k, nullptr, w.e, nullptr, 0);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  kw_chain_kernel<<<(B + CHAIN_THREADS - 1) / CHAIN_THREADS, CHAIN_THREADS, 0, st>>>(n_in, rows, S, B, f, w.ld_k, w.e, w.s, w.carry);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  kw_subblock_kernel<true><<<sgrid, LN_WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, f, m, seg, w.ld_k, w.s, nullptr, w.E, w.E_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  int rc = vtts_resample_run(ctx, 1, OS, x, x_ld, S, n_in, rs_rows, B, (long long)OS * S, max_u, w.u, w.u_ld, st);
  if (rc) return rc;
  const unsigned ptiles = (unsigned)std::max(1LL, (max_peak + PEAK_TILE - 1) / PEAK_TILE);
  peak_kernel<<<dim3(ptiles, B), PEAK_THREADS, 0, st>>>(x, x_ld, w.u, w.u_ld, S, n_in, rows, m, w.part, w.part_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  loudness_gate_kernel<<<B, GATE_THREADS, 0, st>>>(w.E, w.E_ld, S, n_in, rows, m, w.part, w.part_ld, w.peak, out, target, ceiling, gain_db,
                                                   gain_f);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

size_t al(size_t b) { return (b + 255) & ~size_t(255); }

// one-shot buffers in the context workspace: e, s [B][K][4], E [B][K], u [B][4S], tile maxima, gains (g, f)
int ln_oneshot_ws(vtts_ctx* ctx, int B, int S, int m, LnBufs* w, float** gains) {
  const long long K = std::max(1, S / m), U = (long long)OS * S, T = (S + U + PEAK_TILE - 1) / PEAK_TILE;
  const size_t e_b = al((size_t)B * K * 16), E_b = al((size_t)B * K * 4), u_b = al((size_t)B * U * 4), p_b = al((size_t)B * T * 4);
  int rc = ctx->ensure_ws(2 * e_b + E_b + u_b + p_b + al((size_t)B * 8));
  if (rc) return rc;
  char* p = (char*)ctx->ws;
  w->e = (float*)p;
  w->s = (float*)(p + e_b);
  w->E = (float*)(p + 2 * e_b);
  w->u = (float*)(p + 2 * e_b + E_b);
  w->part = (float*)(p + 2 * e_b + E_b + u_b);
  *gains = (float*)(p + 2 * e_b + E_b + u_b + p_b);
  w->ld_k = (int)K;
  w->E_ld = K;
  w->u_ld = U;
  w->part_ld = (int)T;
  w->carry = nullptr;
  w->peak = nullptr;
  return VTTS_OK;
}

// the oversampled index S * OS of a one-shot row must fit an int
constexpr long long S_MAX = INT_MAX / OS;

// the rate and batch shape of a one-shot call of entry point `who`
int ln_args(vtts_ctx* ctx, const char* who, int B, int S, int rate) {
  if (!rate_ok(rate)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rate %d (a multiple of 10 in [8000, 192000])", who, rate);
  return batch_check(ctx, who, B, S, S_MAX);
}

// ... and of a normalize call
int ln_norm_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, float target, float ceiling) {
  const int rc = ln_args(ctx, who, B, S, rate);
  if (rc) return rc;
  if (!(target >= -70.f && target <= 0.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: target %g LUFS (in [-70, 0])", who, (double)target);
  if (!(ceiling == INFINITY || (ceiling >= -20.f && ceiling <= 0.f)))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: ceiling %g dBTP (in [-20, 0], or +inf for none)", who, (double)ceiling);
  return VTTS_OK;
}

int ln_norm_launch(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float target, float ceiling, float* y,
                   float* gain_db, cudaStream_t st) {
  const LnFilter& f = ln_filter(ctx, rate);
  LnBufs w;
  float* gains = nullptr;
  int rc = ln_oneshot_ws(ctx, B, S, rate / 10, &w, &gains);
  if (rc) return rc;
  const long long U = (long long)OS * S;
  // the meter rows land in the e buffer, which the gate no longer reads
  float* g_db = gain_db ? gain_db : gains;
  rc = ln_measure(ctx, f, x, S, S, n_in, nullptr, nullptr, B, S / (rate / 10), U, S + U, w, w.e, target, ceiling, g_db, gains + B, st);
  if (rc) return rc;
  gain_apply_kernel<<<dim3((S + APPLY_THREADS - 1) / APPLY_THREADS, B), APPLY_THREADS, 0, st>>>(x, S, n_in, gains + B, y);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace

size_t vtts_loudness_ws_bytes(int B, int S, int rate) {
  const int m = rate / 10;
  const long long K = std::max(1, S / m), U = (long long)OS * S, T = (S + U + PEAK_TILE - 1) / PEAK_TILE;
  return 2 * al((size_t)B * K * 16) + al((size_t)B * K * 4) + al((size_t)B * U * 4) + al((size_t)B * T * 4) + al((size_t)B * 8);
}

int vtts_loudness_filter(int rate, double* coeffs) {
  if (!rate_ok(rate) || !coeffs) return VTTS_ERR_BAD_ARG;
  ln_design(rate, coeffs);
  return VTTS_OK;
}

int vtts_loudness_launch(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float* out, cudaStream_t st) {
  const LnFilter& f = ln_filter(ctx, rate);
  LnBufs w;
  float* gains = nullptr;
  const int rc = ln_oneshot_ws(ctx, B, S, rate / 10, &w, &gains);
  if (rc) return rc;
  const long long U = (long long)OS * S;
  return ln_measure(ctx, f, x, S, S, n_in, nullptr, nullptr, B, S / (rate / 10), U, S + U, w, out, 0.f, INFINITY, nullptr, nullptr, st);
}

int vtts_loudness(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float* out_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = ln_args(ctx, "loudness", B, S, rate);
  if (rc) return rc;
  if (!x_dev || !out_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "loudness: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return vtts_loudness_launch(ctx, x_dev, n_dev, B, S, rate, out_dev, (cudaStream_t)stream);
}

int vtts_loudness_normalize(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float target, float ceiling,
                            float* y_dev, float* gain_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = ln_norm_args(ctx, "loudness_normalize", B, S, rate, target, ceiling);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "loudness_normalize: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return ln_norm_launch(ctx, x_dev, n_dev, B, S, rate, target, ceiling, y_dev, gain_db_dev, (cudaStream_t)stream);
}

int vtts_loudness_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float* out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = ln_args(ctx, "loudness_host", B, S, rate);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("loudness_host", x, n_in, B, S, out != nullptr);
  if (rc) return rc;
  const size_t o_o = hs.out((size_t)B * 16, out);
  return hs.run([&](cudaStream_t st) { return vtts_loudness_launch(ctx, hs.x(), hs.n(), B, S, rate, hs.dev<float>(o_o), st); });
}

int vtts_loudness_normalize_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float target, float ceiling,
                                 float* y, float* gain_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = ln_norm_args(ctx, "loudness_normalize_host", B, S, rate, target, ceiling);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("loudness_normalize_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_g = hs.out((size_t)B * 4, gain_db), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) {
    return ln_norm_launch(ctx, hs.x(), hs.n(), B, S, rate, target, ceiling, hs.dev<float>(o_y), hs.dev<float>(o_g), st);
  });
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples in P and, in E, the oversampled outputs the running peak covers.
struct vtts_loudness_stream : SampleStream<LnRow, RsRow> {
  using SampleStream::SampleStream;
  int rate = 0, m = 0, hcap = 0, kpush = 0, upitch = 0, ptiles = 0;
  LnBufs w{};
};

int vtts_loudness_stream_lookahead(int rate) {
  if (!rate_ok(rate)) return VTTS_ERR_BAD_ARG;
  return vtts_resample_stream_lookahead(1, OS);
}

int vtts_loudness_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, int max_seconds, vtts_loudness_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "loudness_stream_create", out, true, max_streams, max_chunk_samples);
  if (rc) return rc;
  if (!rate_ok(rate)) return ctx->fail(VTTS_ERR_BAD_ARG, "loudness_stream_create: rate %d (a multiple of 10 in [8000, 192000])", rate);
  if (max_seconds < 1 || max_seconds > (1 << 20))
    return ctx->fail(VTTS_ERR_BAD_ARG, "loudness_stream_create: max_seconds=%d (1..%d)", max_seconds, 1 << 20);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  ln_filter(ctx, rate);
  std::unique_ptr<vtts_loudness_stream> ls(new vtts_loudness_stream(ctx, max_streams, max_chunk_samples, rate / 10));
  ls->rate = rate;
  ls->m = rate / 10;
  ls->hcap = 10 * max_seconds;
  ls->kpush = (ls->m - 1 + max_chunk_samples) / ls->m;            // complete sub-blocks one push can bring
  ls->upitch = OS * max_chunk_samples + 10 * OS + 1;              // oversampled outputs one push can cover
  ls->ptiles = (max_chunk_samples + ls->upitch + PEAK_TILE - 1) / PEAK_TILE;
  const size_t S = max_streams, kp = std::max(1, ls->kpush);
  static_assert(sizeof(LnRow) % 16 == 0 && sizeof(RsRow) % 16 == 0, "table entries keep 16-byte alignment");
  rc = stream_alloc(ctx, "loudness_stream_create", *ls, [&](Arena& a) {
    ls->carve_window(a);
    ls->w.e = a.take<float>(S * kp * 4);
    ls->w.s = a.take<float>(S * kp * 4);
    ls->w.E = a.take<float>(S * ls->hcap);
    ls->w.carry = a.take<float>(S * 4);
    ls->w.peak = a.take<float>(S);
    ls->w.u = a.take<float>(S * ls->upitch);
    ls->w.part = a.take<float>(S * ls->ptiles);
    ls->carve_tables(a);
  });
  if (rc) return rc;
  ls->w.ld_k = (int)kp;
  ls->w.E_ld = ls->hcap;
  ls->w.u_ld = ls->upitch;
  ls->w.part_ld = ls->ptiles;
  *out = ls.release();
  return VTTS_OK;
}

int vtts_loudness_stream_destroy(vtts_ctx* ctx, vtts_loudness_stream* ls) { return stream_destroy(ctx, "loudness_stream_destroy", ls); }

int vtts_loudness_stream_push(vtts_ctx* ctx, vtts_loudness_stream* ls, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                              float* out_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "loudness_stream_push", ls, x_dev && n_new && flags && out_dev);
  if (rc) return rc;
  const int S = ls->S, m = ls->m;
  const SlotState& sl = ls->slots;
  rc = sl.check(ctx, "loudness_stream_push", ls->F, n_new, flags, [&](int s) -> int {
    const long long P1 = ((flags[s] & 1) ? 0 : sl.P[s]) + n_new[s];
    if (P1 / m > ls->hcap)
      return ctx->fail(VTTS_ERR_BAD_ARG, "loudness_stream_push: slot %d would hold %lld samples, more than max_seconds (%d sub-blocks)", s,
                       P1, ls->hcap);
    return VTTS_OK;
  });
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;

  // ---- host bookkeeping: the sub-blocks this push completes and the oversampled outputs whose inputs have all arrived
  // (resample stream schedule of 4 / 1: max(0, 4 P - 40) before END, 4 P with it) ----
  LnRow* rows = ls->rows<0>();
  RsRow* rs = ls->rows<1>();
  const long long half = (long long)vtts_resample_stream_lookahead(1, OS) * OS;
  std::vector<long long> U1(S);
  long long max_k = 0, max_u = 0, max_peak = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    const long long U0 = begin ? 0 : sl.E[s];
    U1[s] = act ? (end ? OS * P1 : std::max(0LL, OS * P1 - half)) : U0;
    LnRow r{};
    r.x0 = P0 - m;
    r.k0 = P0 / m;
    r.nk = (int)(P1 / m - P0 / m);
    r.K = (int)(P1 / m);
    r.xa = m;
    r.nx = act ? n_new[s] : 0;
    r.nu = U1[s] - U0;
    r.begin = begin;
    rows[s] = r;
    rs[s] = RsRow{P0 - m, std::max(0LL, P0 - m), P1, U0, r.nu, r.nu};
    max_k = std::max(max_k, (long long)r.nk);
    max_u = std::max(max_u, r.nu);
    max_peak = std::max(max_peak, r.nx + r.nu);
  }
  if (max_u > ls->upitch || max_k > ls->w.ld_k)
    return ctx->fail(VTTS_ERR_CUDA, "loudness_stream_push: %lld outputs / %lld sub-blocks (internal bound %d / %d)", max_u, max_k, ls->upitch,
                     ls->w.ld_k);

  // ---- device: one table copy, window step, the six measuring launches (seven in all) ----
  rc = ls->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  rc = ln_measure(ctx, ln_filter(ctx, ls->rate), ls->win, ls->cap, ls->cap, nullptr, ls->d_rows<0>(), ls->d_rows<1>(), S, max_k, max_u, max_peak, ls->w,
                  out_dev, 0.f, INFINITY, nullptr, nullptr, st);
  if (rc) return rc;
  ls->slots.commit(n_new, flags, U1.data());
  return VTTS_OK;
}

int vtts_loudness_stream_push_host(vtts_ctx* ctx, vtts_loudness_stream* ls, const float* x, const int32_t* n_new, const uint8_t* flags,
                                   float* out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "loudness_stream_push_host", ls, x && out);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ls->S * ls->F * 4), o_o = hs.out((size_t)ls->S * 16, out);
  return hs.run([&](cudaStream_t st) { return vtts_loudness_stream_push(ctx, ls, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_o), st); });
}
