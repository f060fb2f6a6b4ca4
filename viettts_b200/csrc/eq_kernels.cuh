// The equalizer's filter, kernels and launch sequence (eq.cu states the section form and the block invariant), shared
// by the equalizer and the de-esser's sidechain (deesser.cu).  Internal to each translation unit that includes it.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>

#include "stream_common.cuh"

namespace {
namespace eqk {

constexpr int KMAX = 8;               // sections
constexpr int NS = 2 * KMAX;          // cascade state
constexpr int SEG = 32;               // samples per lane
constexpr int Q = 32 * SEG;           // samples per block (one warp)
constexpr int WARPS = 4;              // blocks per CTA
constexpr long long S_MAX = 1 << 30;  // one-shot row length: int sample indices one block past the row stay exact
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

// the stream row of a slot that holds P0 samples before the push and P1 after it: its window carries the samples from
// P0 - Q on (the incomplete block), it re-runs the blocks from P0's, and it releases every sample the push brings
EqRow eq_stream_row(long long P0, long long P1, int begin) {
  EqRow r{};
  r.x0 = P0 - Q;
  r.r0 = P0;
  r.k0 = P0 / Q;
  r.n = P1;
  r.rn = P1 - P0;
  r.nk = P1 > P0 ? (int)((P1 - 1) / Q - P0 / Q + 1) : 0;
  r.begin = begin;
  return r;
}

// blocks one push of up to F samples can touch
int eq_stream_blocks(int F) { return (Q - 1 + F + Q - 1) / Q; }

}  // namespace eqk
}  // namespace
