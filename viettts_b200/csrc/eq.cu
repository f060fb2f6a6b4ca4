// Equalizer: a cascade of K <= 8 second-order sections over one mono row, fp32 on the device in every vtts_precision
// mode (oracle/eq_oracle.py states it in float64):
//   y = scipy.signal.sosfilt(sos, x) from zero state at sample 0, sos [K][6] = b0 b1 b2 a0 a1 a2;  outputs past n are 0.
//
// Section form.  Every section runs as the trapezoidal (TPT) state-variable filter of its own bilinear transform
// (Simper's linear SVF, the form of the loudness meter's high-pass): with the coefficients normalized by a0,
//   g^2 = (1 + a1 + a2) / (1 - a1 + a2),  k = 2 g (1 - a2) / (1 + a1 + a2)   (both exist for every stable section),
//   n2 = g^2 (b0 - b1 + b2) / c0,  n1 = 2 g (b0 - b2) / c0,  n0 = (b0 + b1 + b2) / c0,  c0 = 1 + a1 + a2,
//   m0 = n2,  m1 = n1 - m0 k,  m2 = n0 - m0,
// derived in double and rounded to fp32 once.  Per sample, state (s1, s2): v3 = x - s2, v1 = d s1 + g d v3,
// v2 = s2 + g d s1 + g^2 d v3 (d = 1 / (1 + g (g + k))), s1 = 2 v1 - s1, s2 = 2 v2 - s2, y = m0 x + m1 v1 + m2 v2.
// Rounded to fp32, direct-form coefficients of a low-frequency section move its poles (a1 = -2 + O(g), a2 = 1 - O(g));
// the state-variable coefficients keep them to fp32 precision.
//
// Invariant (as in loudness.cu and limiter.cu).  Blocks of Q = 1024 samples fixed by absolute sample index.  The
// cascade state entering block k is s_k, s_k+1 = M s_k + e_k, with e_k the block's end state from zero (a fixed fp32
// function of its samples) and M = A^Q (A the 2K x 2K block-lower-triangular one-sample transition of the cascade,
// powered in double and rounded to fp32).  Every output of block k is a fixed fp32 function of s_k and the block's
// samples, so a row gives the same bits alone, in any batch position, in every precision mode and through the stream.
//
// Block kernel.  One warp per (row, block), lane l holding samples [32 l, 32 l + 32) in registers (staged through shared
// memory so the global loads and stores coalesce).  For each section in turn: every lane filters its segment from zero,
// a five-step Hillis-Steele scan with the section's 2 x 2 transitions A_j^(32 2^d) composes the lane end states into
// each lane's entering state (lane 0 enters with zero, or with s_k in the output pass), and every lane re-filters its
// segment from it, which gives the section's exact outputs as the next section's input.  Samples past the row's end
// read as 0; only later samples depend on them, so no lane needs a bound.  The kernel runs twice: from zero (the lane
// holding a complete block's last sample writes e_k) and from s_k (y).
//
// Chain kernel.  One warp per row: the lanes stage 32 blocks' e_k in shared memory, then walk s_k+1 = M s_k + e_k over
// them with lane a < 2K holding state row a and row a of M (the 2K states reach every lane by shuffles), and store the
// 32 entering states.
//
// Stream.  Per slot a window of Q carried samples plus one chunk (the resample stream's window step) and the cascade
// state at the last complete block boundary.  A push re-runs the slot's incomplete block from that boundary and writes
// the outputs of every sample it brought: an IIR filter needs no lookahead.  Every push issues the same four launches.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "stream_common.cuh"

namespace {

constexpr int KMAX = 8;               // sections
constexpr int NS = 2 * KMAX;          // cascade state
constexpr int SEG = 32;               // samples per lane
constexpr int Q = 32 * SEG;           // samples per block (one warp)
constexpr int WARPS = 4;              // blocks per CTA
constexpr int CHAIN_WARPS = 4;        // rows per CTA of the chain kernel
constexpr double POLE_MARGIN = 1e-6;  // every pole radius <= 1 - POLE_MARGIN
constexpr unsigned FULL = 0xffffffffu;

// the fp32 filter, passed by value to every kernel (1.8 KB)
struct EqFilter {
  int K;
  float c[KMAX][6];          // per section: d, g d, g^2 d, m0, m1, m2
  float seg[KMAX][5][4];     // per section: its zero-input transition over 32 * 2^d samples (row-major 2 x 2)
  float blk[NS][NS];         // M = A^Q of the cascade (zero past 2K)
};

struct EqRow {
  long long x0;      // absolute index of input buffer element 0
  long long r0;      // absolute index of output buffer element 0
  long long k0;      // first block processed
  long long n;       // samples of the row so far: inputs at or past n read as 0
  long long rn;      // outputs written: samples [r0, r0 + rn), 0 at or past n
  int nk;            // blocks processed
  int begin;         // the carried state restarts
};
static_assert(sizeof(EqRow) % 16 == 0, "table entries keep 16-byte alignment");

// rows == nullptr: the one-shot row b, n = n_in[b] clamped to [0, S] (or S), outputs [0, S)
__device__ __forceinline__ EqRow eq_row(const EqRow* rows, const int* n_in, int S, int b) {
  if (rows) return rows[b];
  EqRow r;
  r.n = n_in ? min(max(n_in[b], 0), S) : S;
  r.x0 = r.r0 = r.k0 = 0;
  r.rn = S;
  r.nk = (int)((r.n + Q - 1) / Q);
  r.begin = 1;
  return r;
}

// one sample through a section from state (s1, s2); returns y
__device__ __forceinline__ float svf_step(const float (&c)[6], float& s1, float& s2, float x) {
  const float v3 = x - s2;
  const float v1 = fmaf(c[1], v3, c[0] * s1);
  const float v2 = fmaf(c[2], v3, fmaf(c[1], s1, s2));
  s1 = fmaf(2.f, v1, -s1);
  s2 = fmaf(2.f, v2, -s2);
  return fmaf(c[5], v2, fmaf(c[4], v1, c[3] * x));
}

// OUT = false: e_out[row][q][2j, 2j + 1] = section j's end state from zero over complete block k0 + q.  OUT = true:
// lane 0 enters section j with s_in[row][q][2j, 2j + 1] and y gets the cascade's outputs (y may be x: a warp reads
// its whole block before it writes).
template <bool OUT>
__global__ void __launch_bounds__(WARPS * 32) eq_block_kernel(const float* x, long long x_ld, int S, const int* __restrict__ n_in,
                                                              const EqRow* __restrict__ rows, const EqFilter f, int ld_k,
                                                              const float* __restrict__ s_in, float* __restrict__ e_out, float* y,
                                                              long long y_ld) {
  __shared__ float stage[WARPS][Q + 32];   // element i at i + i / 32: conflict-free both ways
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
  const int q = blockIdx.x * WARPS + warp;
  const EqRow r = eq_row(rows, n_in, S, b);
  const long long kq = (r.k0 + q) * Q;
  float* yr = y + (size_t)b * y_ld - r.r0;
  if (q >= r.nk) {                                        // whole warps leave: only warp shuffles below
    if (OUT)                                              // one-shot blocks past the row's end
      for (long long t = max(kq, r.r0) + lane; t < min(kq + Q, r.r0 + r.rn); t += 32) yr[t] = 0.f;
    return;
  }
  float* sh = stage[warp];
  // the block's samples [kq, kq + Q) as offsets m: inputs below nv, outputs in [lo, hi)
  const int nv = (int)min((long long)Q, r.n - kq);
  const float* xb = x + (size_t)b * x_ld + (kq - r.x0);
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    const int m = i * 32 + lane;
    sh[i * 33 + lane] = m < nv ? xb[m] : 0.f;
  }
  __syncwarp();
  float v[SEG];
#pragma unroll
  for (int i = 0; i < SEG; ++i) v[i] = sh[lane * 33 + i];
  const bool complete = nv == Q;
  const float* si = s_in + ((size_t)b * ld_k + q) * NS;
  float* eo = e_out + ((size_t)b * ld_k + q) * NS;
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    if (j >= f.K) break;
    float n1 = 0.f, n2 = 0.f;
    if (OUT && lane == 0) {
      n1 = si[2 * j];
      n2 = si[2 * j + 1];
    }
    float s1 = n1, s2 = n2;
#pragma unroll
    for (int i = 0; i < SEG; ++i) svf_step(f.c[j], s1, s2, v[i]);
    // inclusive scan of u_l = A_j^(32) u_l-1 + (s1, s2)_l
#pragma unroll
    for (int d = 0; d < 5; ++d) {
      const float o1 = __shfl_up_sync(FULL, s1, 1 << d), o2 = __shfl_up_sync(FULL, s2, 1 << d);
      if (lane >= (1 << d)) {
        const float* A = f.seg[j][d];
        const float u1 = fmaf(A[1], o2, fmaf(A[0], o1, s1));
        const float u2 = fmaf(A[3], o2, fmaf(A[2], o1, s2));
        s1 = u1;
        s2 = u2;
      }
    }
    const float p1 = __shfl_up_sync(FULL, s1, 1), p2 = __shfl_up_sync(FULL, s2, 1);
    s1 = lane == 0 ? n1 : p1;
    s2 = lane == 0 ? n2 : p2;
#pragma unroll
    for (int i = 0; i < SEG; ++i) v[i] = svf_step(f.c[j], s1, s2, v[i]);
    if (!OUT && complete && lane == 31) {
      eo[2 * j] = s1;
      eo[2 * j + 1] = s2;
    }
  }
  if (!OUT) return;
  __syncwarp();
#pragma unroll
  for (int i = 0; i < SEG; ++i) sh[lane * 33 + i] = v[i];
  __syncwarp();
  const int lo = (int)max(0LL, r.r0 - kq), hi = (int)min((long long)Q, r.r0 + r.rn - kq);
  float* yb = yr + kq;
#pragma unroll
  for (int i = 0; i < SEG; ++i) {
    const int m = i * 32 + lane;
    if (m >= lo && m < hi) yb[m] = m < nv ? sh[i * 33 + lane] : 0.f;
  }
}

// s_out[row][q] = the state entering block k0 + q: s = M s + e over the row's complete blocks, from carry[row] (unless
// the row begins) or zero; the state at the last complete block boundary goes back to carry.  Lane a < 2K carries state
// row a and row a of M; each step takes the 2K states by shuffles, in column order.
__global__ void __launch_bounds__(CHAIN_WARPS * 32) eq_chain_kernel(const int* __restrict__ n_in, const EqRow* __restrict__ rows, int S,
                                                                    int B, const EqFilter f, int ld_k, const float* __restrict__ e,
                                                                    float* __restrict__ s_out, float* __restrict__ carry) {
  __shared__ float stage[CHAIN_WARPS][32 * NS];            // 32 blocks' e, then their entering states
  __shared__ float msh[NS * NS];
  const float* mp = &f.blk[0][0];
#pragma unroll
  for (int i = 0; i < NS * NS; ++i)                        // static indices keep f in the parameter bank
    if (i % (CHAIN_WARPS * 32) == (int)threadIdx.x) msh[i] = mp[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * CHAIN_WARPS + warp;
  if (b >= B) return;                                     // whole warps leave
  const EqRow r = eq_row(rows, n_in, S, b);
  const int n = 2 * f.K;
  const bool own = lane < n;
  float m[NS];
#pragma unroll
  for (int c = 0; c < NS; ++c) m[c] = own ? msh[lane * NS + c] : 0.f;
  float s = (own && carry && !r.begin) ? carry[(size_t)b * NS + lane] : 0.f;
  const float* er = e + (size_t)b * ld_k * NS;
  float* so = s_out + (size_t)b * ld_k * NS;
  float* sh = stage[warp];
  for (int q0 = 0; q0 < r.nk; q0 += 32) {
    const int cnt = min(32, r.nk - q0);
    // the complete blocks lead: block k0 + q is complete while q < floor(n / Q) - k0
    const int ncomp = (int)max(0LL, min((long long)cnt, r.n / Q - r.k0 - q0));
    for (int i = lane; i < ncomp * NS; i += 32) sh[i] = er[(size_t)q0 * NS + i];
    __syncwarp();
    for (int i = 0; i < cnt; ++i) {
      const float ev = own ? sh[i * NS + lane] : 0.f;
      if (own) sh[i * NS + lane] = s;
      if (i < ncomp) {
        float acc = ev;
#pragma unroll
        for (int c = 0; c < NS; ++c) {
          if (c >= n) break;
          acc = fmaf(m[c], __shfl_sync(FULL, s, c), acc);
        }
        s = own ? acc : 0.f;
      }
    }
    __syncwarp();
    for (int i = lane; i < cnt * NS; i += 32) so[(size_t)q0 * NS + i] = sh[i];
    __syncwarp();
  }
  if (carry && own) carry[(size_t)b * NS + lane] = s;
}

// ---- the filter on the host ---------------------------------------------------------------------------------------

// largest pole radius of z^2 + a1 z + a2
double pole_radius(double a1, double a2) {
  const double disc = a1 * a1 - 4.0 * a2;
  if (disc < 0.0) return std::sqrt(a2);
  const double r = std::sqrt(disc);
  return std::max(std::fabs(-a1 + r), std::fabs(-a1 - r)) * 0.5;
}

// p = d, g d, g^2 d, m0, m1, m2 of section `row` (b0 b1 b2 a0 a1 a2) in double; false unless it is finite, a0 != 0 and
// strictly stable with every pole radius <= 1 - POLE_MARGIN
bool svf_params(const double* row, double* p) {
  for (int i = 0; i < 6; ++i)
    if (!std::isfinite(row[i])) return false;
  if (row[3] == 0.0) return false;
  const double b0 = row[0] / row[3], b1 = row[1] / row[3], b2 = row[2] / row[3], a1 = row[4] / row[3], a2 = row[5] / row[3];
  if (!(std::fabs(a2) < 1.0 && std::fabs(a1) < 1.0 + a2) || pole_radius(a1, a2) > 1.0 - POLE_MARGIN) return false;
  const double c0 = 1.0 + a1 + a2, g = std::sqrt(c0 / (1.0 - a1 + a2)), k = 2.0 * g * (1.0 - a2) / c0;
  const double n2 = g * g * (b0 - b1 + b2) / c0, n1 = 2.0 * g * (b0 - b2) / c0, n0 = (b0 + b1 + b2) / c0;
  const double d = 1.0 / (1.0 + g * (g + k));
  const double q[6] = {d, g * d, g * g * d, n2, n1 - n2 * k, n0 - n2};
  for (int i = 0; i < 6; ++i) {
    if (!std::isfinite(q[i])) return false;
    p[i] = q[i];
  }
  return true;
}

// one sample through the cascade in double (the kernels' svf_step)
void cascade_step(const double (*p)[6], int K, double* s, double x) {
  for (int j = 0; j < K; ++j) {
    const double* c = p[j];
    double& s1 = s[2 * j];
    double& s2 = s[2 * j + 1];
    const double v3 = x - s2, v1 = c[0] * s1 + c[1] * v3, v2 = s2 + c[1] * s1 + c[2] * v3;
    s1 = 2.0 * v1 - s1;
    s2 = 2.0 * v2 - s2;
    x = c[3] * x + c[4] * v1 + c[5] * v2;
  }
}

int eq_filter(vtts_ctx* ctx, const char* who, const double* sos, int K, EqFilter* f) {
  if (!sos) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null sos", who);
  if (K < 1 || K > KMAX) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: K=%d sections (1..%d)", who, K, KMAX);
  double p[KMAX][6];
  for (int j = 0; j < K; ++j)
    if (!svf_params(sos + 6 * j, p[j]))
      return ctx->fail(VTTS_ERR_BAD_ARG,
                       "%s: section %d (%g %g %g %g %g %g) must be finite with a0 != 0 and strictly stable (pole radius <= 1 - %g)", who,
                       j, sos[6 * j], sos[6 * j + 1], sos[6 * j + 2], sos[6 * j + 3], sos[6 * j + 4], sos[6 * j + 5], POLE_MARGIN);
  std::memset(f, 0, sizeof(*f));
  f->K = K;
  const int n = 2 * K;
  // zero-input one-sample transition of the cascade: column c = the state after one step from unit state c
  std::vector<double> A(n * n), P(n * n);
  for (int c = 0; c < n; ++c) {
    double s[NS] = {};
    s[c] = 1.0;
    cascade_step(p, K, s, 0.0);
    for (int i = 0; i < n; ++i) A[i * n + c] = s[i];
  }
  for (int j = 0; j < K; ++j) {
    for (int i = 0; i < 6; ++i) f->c[j][i] = (float)p[j][i];
    const double Aj[4] = {A[(2 * j) * n + 2 * j], A[(2 * j) * n + 2 * j + 1], A[(2 * j + 1) * n + 2 * j], A[(2 * j + 1) * n + 2 * j + 1]};
    double Pj[4];
    for (int d = 0; d < 5; ++d) {
      vtts_mat_pow(Aj, (long long)SEG << d, Pj, 2);
      for (int i = 0; i < 4; ++i) f->seg[j][d][i] = (float)Pj[i];
    }
  }
  vtts_mat_pow(A.data(), Q, P.data(), n);
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < n; ++c) f->blk[i][c] = (float)P[i * n + c];
  return VTTS_OK;
}

// the three launches of a call: zero-state pass, chain, output pass
int eq_run(vtts_ctx* ctx, const EqFilter& f, const float* x, long long x_ld, int S, const int* n_in, const EqRow* rows, int B, long long max_k,
           int ld_k, float* e, float* s, float* carry, float* y, long long y_ld, cudaStream_t st) {
  const dim3 grid((unsigned)std::max(1LL, (max_k + WARPS - 1) / WARPS), B);
  eq_block_kernel<false><<<grid, WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, f, ld_k, nullptr, e, nullptr, 0);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  eq_chain_kernel<<<(B + CHAIN_WARPS - 1) / CHAIN_WARPS, CHAIN_WARPS * 32, 0, st>>>(n_in, rows, S, B, f, ld_k, e, s, carry);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  eq_block_kernel<true><<<grid, WARPS * 32, 0, st>>>(x, x_ld, S, n_in, rows, f, ld_k, s, nullptr, y, y_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

size_t al(size_t b) { return (b + 255) & ~size_t(255); }

int eq_check(vtts_ctx* ctx, const char* who, int B, int S) {
  if (B < 1 || B > 65535 || S < 1 || S > (1 << 30))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: B=%d S=%d (1..65535, 1..2^30)", who, B, S);
  return VTTS_OK;
}

// ---- the designer ---------------------------------------------------------------------------------------------------

void put(double* row, double b0, double b1, double b2, double a0, double a1, double a2) {
  const double v[6] = {b0 / a0, b1 / a0, b2 / a0, 1.0, a1 / a0, a2 / a0};
  std::memcpy(row, v, sizeof(v));
}

}  // namespace

int vtts_eq_design(int kind, int rate, double f0, double q, double gain_db, int order, double* sos, int* n_sections) {
  if (!sos || !n_sections) return VTTS_ERR_BAD_ARG;
  if (rate < 8000 || rate > 192000 || !(f0 >= 10.0 && f0 <= 0.45 * rate)) return VTTS_ERR_BAD_ARG;
  const double pi = 3.14159265358979323846;
  const double w0 = 2.0 * pi * f0 / rate, cw = std::cos(w0), sw = std::sin(w0);
  const bool gain_ok = gain_db >= -24.0 && gain_db <= 24.0, q_ok = q >= 0.1 && q <= 30.0;
  const double A = std::pow(10.0, gain_db / 40.0);
  switch (kind) {
    case VTTS_EQ_HIGHPASS:
    case VTTS_EQ_LOWPASS: {
      // Butterworth: pairs s^2 + 2 sin(pi (2i + 1) / 2N) s + 1 and, for odd N, s + 1, through the bilinear transform
      // prewarped to f0 (s = (z - 1) / (K (z + 1)), K = tan(pi f0 / rate))
      if (order < 1 || order > 8) return VTTS_ERR_BAD_ARG;
      const bool hp = kind == VTTS_EQ_HIGHPASS;
      const double K = std::tan(pi * f0 / rate), K2 = K * K;
      int j = 0;
      for (int i = 0; i < order / 2; ++i, ++j) {
        const double z2 = 2.0 * std::sin(pi * (2 * i + 1) / (2.0 * order));
        const double a0 = 1.0 + z2 * K + K2, a1 = 2.0 * (K2 - 1.0), a2 = 1.0 - z2 * K + K2;
        if (hp)
          put(sos + 6 * j, 1.0, -2.0, 1.0, a0, a1, a2);
        else
          put(sos + 6 * j, K2, 2.0 * K2, K2, a0, a1, a2);
      }
      if (order % 2) {
        if (hp)
          put(sos + 6 * j, 1.0, -1.0, 0.0, 1.0 + K, K - 1.0, 0.0);
        else
          put(sos + 6 * j, K, K, 0.0, 1.0 + K, K - 1.0, 0.0);
        ++j;
      }
      *n_sections = j;
      return VTTS_OK;
    }
    case VTTS_EQ_LOWSHELF:
    case VTTS_EQ_HIGHSHELF: {
      // RBJ Audio EQ Cookbook shelves, q = the shelf slope S in (0, 1]
      if (!(q > 0.0 && q <= 1.0) || !gain_ok) return VTTS_ERR_BAD_ARG;
      const double alpha = sw / 2.0 * std::sqrt((A + 1.0 / A) * (1.0 / q - 1.0) + 2.0), ra = 2.0 * std::sqrt(A) * alpha;
      if (kind == VTTS_EQ_LOWSHELF)
        put(sos, A * ((A + 1) - (A - 1) * cw + ra), 2 * A * ((A - 1) - (A + 1) * cw), A * ((A + 1) - (A - 1) * cw - ra),
            (A + 1) + (A - 1) * cw + ra, -2 * ((A - 1) + (A + 1) * cw), (A + 1) + (A - 1) * cw - ra);
      else
        put(sos, A * ((A + 1) + (A - 1) * cw + ra), -2 * A * ((A - 1) + (A + 1) * cw), A * ((A + 1) + (A - 1) * cw - ra),
            (A + 1) - (A - 1) * cw + ra, 2 * ((A - 1) - (A + 1) * cw), (A + 1) - (A - 1) * cw - ra);
      *n_sections = 1;
      return VTTS_OK;
    }
    case VTTS_EQ_PEAKING: {
      if (!q_ok || !gain_ok) return VTTS_ERR_BAD_ARG;
      const double alpha = sw / (2.0 * q);
      put(sos, 1.0 + alpha * A, -2.0 * cw, 1.0 - alpha * A, 1.0 + alpha / A, -2.0 * cw, 1.0 - alpha / A);
      *n_sections = 1;
      return VTTS_OK;
    }
    case VTTS_EQ_NOTCH: {
      if (!q_ok) return VTTS_ERR_BAD_ARG;
      const double alpha = sw / (2.0 * q);
      put(sos, 1.0, -2.0 * cw, 1.0, 1.0 + alpha, -2.0 * cw, 1.0 - alpha);
      *n_sections = 1;
      return VTTS_OK;
    }
    default:
      return VTTS_ERR_BAD_ARG;
  }
}

int vtts_eq(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const double* sos, int K, float* y_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  EqFilter f;
  int rc = eq_check(ctx, "eq", B, S);
  if (!rc) rc = eq_filter(ctx, "eq", sos, K, &f);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "eq: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const int nb = (S + Q - 1) / Q;
  const size_t es_b = al((size_t)B * nb * NS * 4);
  rc = ctx->ensure_ws(2 * es_b);
  if (rc) return rc;
  float* e = (float*)ctx->ws;
  float* s = (float*)((char*)ctx->ws + es_b);
  return eq_run(ctx, f, x_dev, S, S, n_dev, nullptr, B, nb, nb, e, s, nullptr, y_dev, S, (cudaStream_t)stream);
}

int vtts_eq_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const double* sos, int K, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  EqFilter f;
  int rc = eq_check(ctx, "eq_host", B, S);
  if (!rc) rc = eq_filter(ctx, "eq_host", sos, K, &f);
  if (!rc) rc = host_lengths_check(ctx, "eq_host", n_in, B, S);
  if (rc) return rc;
  if (!x || !y) return ctx->fail(VTTS_ERR_BAD_ARG, "eq_host: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t x_b = (size_t)B * S * 4, n_b = (size_t)B * 4;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, x_b), o_n = hs.in(n_in, n_b), o_y = hs.out(x_b);
  rc = hs.upload();
  if (!rc) rc = vtts_eq(ctx, hs.dev<const float>(o_x), n_in ? hs.dev<const int32_t>(o_n) : nullptr, B, S, sos, K, hs.dev<float>(o_y), hs.st);
  if (!rc) rc = hs.fetch(o_y, y, x_b);
  return rc ? rc : hs.finish();
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and released in E (the same: no lookahead).
struct vtts_eq_stream : SampleStream<EqRow> {
  using SampleStream::SampleStream;
  EqFilter f{};
  int ld_k = 0;
  float *e = nullptr, *s = nullptr, *carry = nullptr;
};

int vtts_eq_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, const double* sos, int K, vtts_eq_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!out) return ctx->fail(VTTS_ERR_BAD_ARG, "eq_stream_create: null output pointer");
  *out = nullptr;
  if (max_streams < 1 || max_streams > 65535 || max_chunk_samples < 1 || max_chunk_samples > (1 << 22))
    return ctx->fail(VTTS_ERR_BAD_ARG, "eq_stream_create: max_streams=%d max_chunk_samples=%d (1..65535, 1..%d)", max_streams,
                     max_chunk_samples, 1 << 22);
  EqFilter f;
  int rc = eq_filter(ctx, "eq_stream_create", sos, K, &f);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_eq_stream> es(new vtts_eq_stream(ctx, max_streams, max_chunk_samples, Q));
  es->f = f;
  es->ld_k = (Q - 1 + max_chunk_samples + Q - 1) / Q;     // blocks one push can touch
  const size_t S = max_streams;
  rc = stream_alloc(ctx, "eq_stream_create", *es, [&](Arena& a) {
    es->carve_window(a);
    es->e = a.take<float>(S * es->ld_k * NS);
    es->s = a.take<float>(S * es->ld_k * NS);
    es->carry = a.take<float>(S * NS);
    es->carve_tables(a);
  });
  if (rc) return rc;
  *out = es.release();
  return VTTS_OK;
}

int vtts_eq_stream_destroy(vtts_ctx* ctx, vtts_eq_stream* es) { return stream_destroy(ctx, "eq_stream_destroy", es); }

int vtts_eq_stream_push(vtts_ctx* ctx, vtts_eq_stream* es, const float* x_dev, const int32_t* n_new, const uint8_t* flags, float* y_dev,
                        int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "eq_stream_push", es, x_dev && n_new && flags && y_dev && n_out);
  if (rc) return rc;
  const SlotState& sl = es->slots;
  rc = sl.check(ctx, "eq_stream_push", es->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int S = es->S;

  // ---- host bookkeeping: every sample is released in the push that brings it ----
  EqRow* rows = es->rows<0>();
  std::vector<long long> E1(S);
  long long max_k = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    EqRow r{};
    r.x0 = P0 - Q;
    r.r0 = P0;
    r.k0 = P0 / Q;
    r.n = P1;
    r.rn = P1 - P0;
    r.nk = P1 > P0 ? (int)((P1 - 1) / Q - P0 / Q + 1) : 0;
    r.begin = begin;
    rows[s] = r;
    E1[s] = P1;
    n_out[s] = (int32_t)(P1 - P0);
    max_k = std::max(max_k, (long long)r.nk);
  }
  if (max_k > es->ld_k) return ctx->fail(VTTS_ERR_CUDA, "eq_stream_push: %lld blocks (internal bound %d)", max_k, es->ld_k);

  // ---- device: one table copy, window step, the three filter launches (four in all) ----
  rc = es->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  rc = eq_run(ctx, es->f, es->win, es->cap, es->cap, nullptr, es->d_rows<0>(), S, max_k, es->ld_k, es->e, es->s, es->carry, y_dev, es->F, st);
  if (rc) return rc;
  es->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_eq_stream_push_host(vtts_ctx* ctx, vtts_eq_stream* es, const float* x, const int32_t* n_new, const uint8_t* flags, float* y,
                             int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "eq_stream_push_host", es, x && y);
  if (rc) return rc;
  const size_t b = (size_t)es->S * es->F * 4;
  return stream_push_host(ctx, x, b, y, b, [&](const float* x_dev, float* y_dev, cudaStream_t st) {
    return vtts_eq_stream_push(ctx, es, x_dev, n_new, flags, y_dev, n_out, st);
  });
}
