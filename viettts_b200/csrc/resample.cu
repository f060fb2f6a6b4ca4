// Rational-rate resampling of synthesized audio: exactly scipy.signal.resample_poly(x, up, down) with its defaults
// (Kaiser beta = 5 low-pass of 2 * half + 1 taps, half = 10 * max(up, down), zero padding), in fp32 on the device.
//
// Filter.  Designed on the host in double precision (Kaiser window through an I0 series, cutoff 1 / max(up, down), unit
// DC gain, times up), rounded to fp32 once and cached in the context per reduced ratio.  Polyphase layout [phase][tap]
// with T = ceil((2 * half + 1) / up) taps per phase: output m has j = m * down + half, phase p = j mod up and top input
// it = floor(j / up); tap t of phase p multiplies input it - (T - 1) + t and holds h[p + (T - 1 - t) * up] (0 past
// 2 * half).  Every output is therefore the same T-term fp32 FMA sum in ascending input index, a function of m alone:
// the one-shot call and every push pattern of the stream produce the same bits.  up == down is a copy (T = 1, h = 1).
//
// Windows.  A CTA computes a tile of consecutive outputs of one row; it stages the filter and the input span the tile
// reads in shared memory.  Per-row bounds (RsRow) place the row's buffer in absolute time: element 0 is input x0, inputs
// outside [lo, hi) read as zero, outputs m0 .. m0 + n_calc - 1 are computed and written from the row's start and the
// outputs after them up to n_out are written as zero.  Absolute input and output indices are 64-bit: m * down + half
// passes 2^31 after about 4.9 M input samples at 16000 -> 11025.
//
// Stream.  Per slot a window of K + F inputs (K = T - 1 carried, F = max chunk); one prep launch per push moves the last
// K inputs of the previous push to the front and copies the new ones after them, then resample_kernel runs on the
// windows with bounds built on the host.
#include <algorithm>
#include <cmath>

#include "stream_common.cuh"

namespace {

constexpr int RS_MAX_FACTOR = 1024;   // largest reduced up / down
constexpr int RS_THREADS = 256;
constexpr int RS_SMEM_MAX = 227 * 1024;

struct RsRatio {
  int up, down, half, T;
};

long long gcd_ll(long long a, long long b) {
  while (b) {
    long long t = a % b;
    a = b;
    b = t;
  }
  return a;
}

// 0, or VTTS_ERR_BAD_ARG for a non-positive rate or a reduced ratio past RS_MAX_FACTOR
int rs_ratio(int in_rate, int out_rate, RsRatio* r) {
  if (in_rate <= 0 || out_rate <= 0) return VTTS_ERR_BAD_ARG;
  const long long g = gcd_ll(in_rate, out_rate);
  r->up = (int)(out_rate / g);
  r->down = (int)(in_rate / g);
  if (r->up > RS_MAX_FACTOR || r->down > RS_MAX_FACTOR) return VTTS_ERR_BAD_ARG;
  r->half = r->up == r->down ? 0 : 10 * std::max(r->up, r->down);
  r->T = (2 * r->half + r->up) / r->up;   // ceil((2 * half + 1) / up)
  return VTTS_OK;
}

double bessel_i0(double x) {
  double sum = 1.0, term = 1.0;
  const double q = 0.25 * x * x;
  for (int k = 1; k < 500; ++k) {
    term *= q / ((double)k * k);
    sum += term;
    if (term < 1e-17 * sum) break;
  }
  return sum;
}

// h[0 .. 2 * half]: firwin(2 * half + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up
std::vector<double> rs_design(const RsRatio& r) {
  if (r.half == 0) return {1.0};
  const int L = 2 * r.half + 1;
  const double fc = 1.0 / std::max(r.up, r.down), beta = 5.0, i0b = bessel_i0(beta), pi = 3.14159265358979323846;
  std::vector<double> h(L);
  double sum = 0.0;
  for (int k = 0; k < L; ++k) {
    const double a = (double)(k - r.half) / r.half;
    const double w = bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - a * a))) / i0b;
    const double t = fc * (k - r.half);
    const double y = pi * (t == 0.0 ? 1e-20 : t);
    h[k] = fc * (std::sin(y) / y) * w;
    sum += h[k];
  }
  for (int k = 0; k < L; ++k) h[k] = h[k] / sum * r.up;
  return h;
}

// rows == nullptr: the one-shot bounds of row b, inputs [0, n_b) with n_b = n_in[b] (or S_in), S_out outputs of which
// the first ceil(n_b * up / down) are computed
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const float* __restrict__ x, long long x_ld, int S_in,
                                                              const int* __restrict__ n_in, const RsRow* __restrict__ rows,
                                                              const float* __restrict__ taps, int up, int down, int half, int T,
                                                              long long S_out, int TM, float* __restrict__ y, long long y_ld) {
  extern __shared__ float rs_smem[];
  const int b = blockIdx.y, tid = threadIdx.x;
  RsRow r;
  if (rows) {
    r = rows[b];
  } else {
    const long long n = n_in ? (long long)min(max(n_in[b], 0), S_in) : (long long)S_in;
    r.x0 = 0; r.lo = 0; r.hi = n; r.m0 = 0; r.n_out = S_out;
    r.n_calc = min(S_out, (n * up + down - 1) / down);
  }
  const long long t0 = (long long)blockIdx.x * TM;
  if (t0 >= r.n_out) return;
  const int cnt = (int)min((long long)TM, r.n_out - t0);
  const int cc = (int)max(0LL, min((long long)cnt, r.n_calc - t0));
  float* yr = y + (size_t)b * y_ld + t0;
  for (int q = cc + tid; q < cnt; q += RS_THREADS) yr[q] = 0.f;
  if (cc == 0) return;

  const long long mA = r.m0 + t0;
  const long long i_lo = (mA * down + half) / up - (T - 1);
  const long long i_hi = ((mA + cc - 1) * down + half) / up;
  const int span = (int)(i_hi - i_lo + 1);
  float* hs = rs_smem;
  float* xs = rs_smem + up * T;
  for (int e = tid; e < up * T; e += RS_THREADS) hs[e] = taps[e];
  const long long lo = max(r.lo, r.x0), hi = r.hi;
  const float* xr = x + (size_t)b * x_ld;
  for (int e = tid; e < span; e += RS_THREADS) {
    const long long i = i_lo + e;
    xs[e] = (i >= lo && i < hi) ? __ldg(xr + (i - r.x0)) : 0.f;
  }
  __syncthreads();
  for (int q = tid; q < cc; q += RS_THREADS) {
    const long long j = (mA + q) * down + half;
    const long long it = j / up;
    const int p = (int)(j - it * up);
    const float* xq = xs + (it - (T - 1) - i_lo);
    const float* hq = hs + p * T;
    float acc = xq[0] * hq[0];
#pragma unroll 4
    for (int t = 1; t < T; ++t) acc = fmaf(xq[t], hq[t], acc);
    yr[q] = acc;
  }
}

// per slot: tbl[2s] = inputs of the previous push (its window tail [shift, shift + K) moves to [0, K)), tbl[2s + 1] =
// new inputs to copy to [K, K + n)
__global__ void __launch_bounds__(RS_THREADS) resample_prep_kernel(float* __restrict__ win, int cap, int K, const int* __restrict__ tbl,
                                                                   const float* __restrict__ x, int F) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int shift = tbl[2 * b], n = tbl[2 * b + 1];
  float* w = win + (size_t)b * cap;
  if (shift > 0) {
    // source and destination overlap when the push was shorter than the carry: each block of 1024 values is read
    // completely before it is written, in ascending order (the destination lies before the source)
    constexpr int U = 4;
    for (int i0 = 0; i0 < K; i0 += RS_THREADS * U) {
      float v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * RS_THREADS + tid;
        if (i < K) v[u] = w[shift + i];
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * RS_THREADS + tid;
        if (i < K) w[i] = v[u];
      }
      __syncthreads();
    }
  }
  const float* src = x + (size_t)b * F;
  for (int i = tid; i < n; i += RS_THREADS) w[K + i] = src[i];
}

// tile of outputs per CTA: 1024 unless the filter plus the input span do not fit in shared memory
int rs_tile(const RsRatio& r, size_t* smem) {
  int TM = 1024;
  auto bytes = [&](int tm) { return ((size_t)r.up * r.T + ((size_t)(tm - 1) * r.down + r.up - 1) / r.up + r.T) * sizeof(float); };
  while (TM > 1 && bytes(TM) > (size_t)RS_SMEM_MAX) TM /= 2;
  *smem = bytes(TM);
  return TM;
}

// the context's fp32 polyphase filter of ratio r (designed and uploaded at the first use)
int rs_filter(vtts_ctx* ctx, const RsRatio& r, const float** out) {
  for (const auto& f : ctx->rs_filters)
    if (f.up == r.up && f.down == r.down) {
      *out = f.taps;
      return VTTS_OK;
    }
  const std::vector<double> h = rs_design(r);
  std::vector<float> pp((size_t)r.up * r.T, 0.f);
  for (int p = 0; p < r.up; ++p)
    for (int t = 0; t < r.T; ++t) {
      const long long k = p + (long long)(r.T - 1 - t) * r.up;
      if (k <= 2 * r.half) pp[(size_t)p * r.T + t] = (float)h[k];
    }
  float* d = nullptr;
  VTTS_CUDA(cudaMalloc(&d, pp.size() * sizeof(float)));
  cudaError_t e = cudaMemcpy(d, pp.data(), pp.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d);
    return ctx->fail(VTTS_ERR_CUDA, "resample: filter upload: %s", cudaGetErrorString(e));
  }
  ctx->rs_filters.push_back({r.up, r.down, d});
  *out = d;
  return VTTS_OK;
}

int rs_launch(vtts_ctx* ctx, const RsRatio& r, const float* taps, const float* x, long long x_ld, int S_in, const int* n_in,
              const RsRow* rows, int B, long long S_out, long long max_out, float* y, long long y_ld, cudaStream_t st) {
  size_t smem = 0;
  const int TM = rs_tile(r, &smem);
  static bool attr_set[64] = {};
  if (ctx->device < 64 && !attr_set[ctx->device]) {
    VTTS_CUDA(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RS_SMEM_MAX));
    attr_set[ctx->device] = true;
  }
  const long long tiles = std::max(1LL, (max_out + TM - 1) / TM);
  resample_kernel<<<dim3((unsigned)tiles, B), RS_THREADS, smem, st>>>(x, x_ld, S_in, n_in, rows, taps, r.up, r.down, r.half, r.T, S_out, TM,
                                                                     y, y_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

}  // namespace

int vtts_stream_window_prep(vtts_ctx* ctx, float* win, int cap, int K, const int* tbl, const float* x, int F, int S, cudaStream_t st) {
  resample_prep_kernel<<<S, RS_THREADS, 0, st>>>(win, cap, K, tbl, x, F);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

int vtts_resample_run(vtts_ctx* ctx, int in_rate, int out_rate, const float* x, long long x_ld, int S_in, const int* n_in,
                      const RsRow* rows, int B, long long S_out, long long max_out, float* y, long long y_ld, cudaStream_t st) {
  RsRatio r;
  if (rs_ratio(in_rate, out_rate, &r)) return ctx->fail(VTTS_ERR_BAD_ARG, "resample: rates %d -> %d", in_rate, out_rate);
  const float* taps = nullptr;
  int rc = rs_filter(ctx, r, &taps);
  if (rc) return rc;
  return rs_launch(ctx, r, taps, x, x_ld, S_in, n_in, rows, B, S_out, max_out, y, y_ld, st);
}

void vtts_resample_free(vtts_ctx* ctx) {
  for (auto& f : ctx->rs_filters) cudaFree(f.taps);
  ctx->rs_filters.clear();
}

int vtts_resample_filter(int in_rate, int out_rate, double* taps, int capacity) {
  RsRatio r;
  if (rs_ratio(in_rate, out_rate, &r)) return VTTS_ERR_BAD_ARG;
  const std::vector<double> h = rs_design(r);
  if (taps && capacity >= (int)h.size()) std::copy(h.begin(), h.end(), taps);
  return (int)h.size();
}

namespace {

// the rates and batch shape of a one-shot call of entry point `who`
int rs_args(vtts_ctx* ctx, const char* who, int B, int S_in, int in_rate, int out_rate, RsRatio* r) {
  if (rs_ratio(in_rate, out_rate, r))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rates %d -> %d (positive, reduced ratio up / down <= %d)", who, in_rate, out_rate, RS_MAX_FACTOR);
  return batch_check(ctx, who, B, S_in, S_ANY);
}

long long rs_out_samples(const RsRatio& r, int S_in) { return ceil_div((long long)S_in * r.up, r.down); }

int rs_oneshot(vtts_ctx* ctx, const RsRatio& r, const float* x, const int32_t* n_in, int B, int S_in, float* y, cudaStream_t st) {
  const float* taps = nullptr;
  const int rc = rs_filter(ctx, r, &taps);
  if (rc) return rc;
  const long long S_out = rs_out_samples(r, S_in);
  return rs_launch(ctx, r, taps, x, S_in, S_in, n_in, nullptr, B, S_out, S_out, y, S_out, st);
}

}  // namespace

int vtts_resample(vtts_ctx* ctx, const float* x_dev, const int32_t* n_in_dev, int B, int S_in, int in_rate, int out_rate, float* y_dev,
                  void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  RsRatio r;
  const int rc = rs_args(ctx, "resample", B, S_in, in_rate, out_rate, &r);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "resample: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return rs_oneshot(ctx, r, x_dev, n_in_dev, B, S_in, y_dev, (cudaStream_t)stream);
}

int vtts_resample_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S_in, int in_rate, int out_rate, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  RsRatio r;
  int rc = rs_args(ctx, "resample_host", B, S_in, in_rate, out_rate, &r);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("resample_host", x, n_in, B, S_in, y != nullptr);
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * rs_out_samples(r, S_in) * 4, y);
  return hs.run([&](cudaStream_t st) { return rs_oneshot(ctx, r, hs.x(), hs.n(), B, S_in, hs.dev<float>(o_y), st); });
}

// ---- stream ---------------------------------------------------------------------------------------------------
struct vtts_resample_stream : SampleStream<RsRow> {
  using SampleStream::SampleStream;
  RsRatio r{};
  int out_pitch = 0;
  const float* taps = nullptr;
};

int vtts_resample_stream_lookahead(int in_rate, int out_rate) {
  RsRatio r;
  if (rs_ratio(in_rate, out_rate, &r)) return VTTS_ERR_BAD_ARG;
  return r.half / r.up;
}

int vtts_resample_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int in_rate, int out_rate,
                                vtts_resample_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "resample_stream_create", out, out_pitch != nullptr, max_streams, max_chunk_samples);
  if (rc) return rc;
  RsRatio r;
  if (rs_ratio(in_rate, out_rate, &r))
    return ctx->fail(VTTS_ERR_BAD_ARG, "resample_stream_create: rates %d -> %d (positive, reduced ratio up / down <= %d)", in_rate, out_rate,
                     RS_MAX_FACTOR);
  // outputs per push: fewer than (n_new * up + half + 1) / down + 1 (see the schedule in vtts_resample_stream_push)
  const long long pitch = ceil_div((long long)max_chunk_samples * r.up + r.half + 1, r.down);
  if (pitch > (1LL << 30)) return ctx->fail(VTTS_ERR_BAD_ARG, "resample_stream_create: %lld outputs per push", pitch);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const float* taps = nullptr;
  rc = rs_filter(ctx, r, &taps);
  if (rc) return rc;
  std::unique_ptr<vtts_resample_stream> rs(new vtts_resample_stream(ctx, max_streams, max_chunk_samples, r.T - 1));
  rs->r = r;
  rs->out_pitch = (int)pitch;
  rs->taps = taps;
  rc = stream_alloc(ctx, "resample_stream_create", *rs, [&](Arena& a) {
    rs->carve_window(a);
    rs->carve_tables(a);
  });
  if (rc) return rc;
  *out_pitch = rs->out_pitch;
  *out = rs.release();
  return VTTS_OK;
}

int vtts_resample_stream_destroy(vtts_ctx* ctx, vtts_resample_stream* rs) { return stream_destroy(ctx, "resample_stream_destroy", rs); }

int vtts_resample_stream_push(vtts_ctx* ctx, vtts_resample_stream* rs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                              float* y_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "resample_stream_push", rs, x_dev && n_new && flags && y_dev && n_out);
  if (!rc) rc = rs->slots.check(ctx, "resample_stream_push", rs->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = rs->S;
  const RsRatio& r = rs->r;
  const SlotState& sl = rs->slots;

  // ---- host bookkeeping: an output is emitted once every input it reads has arrived, i.e. after P inputs (before END)
  // the slot has emitted min(ceil(P * up / down), max(0, floor((P * up - 1 - half) / down) + 1)) outputs ----
  RsRow* rows = rs->rows<0>();
  std::vector<long long> E1(S);
  long long max_out = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
    const long long P0 = begin ? 0 : sl.P[s], E0 = begin ? 0 : sl.E[s], P1 = P0 + n_new[s];
    long long e = E0;
    if (act) {
      const long long total = ceil_div(P1 * r.up, r.down), v = P1 * r.up - 1 - r.half;
      e = end ? total : std::min(total, v < 0 ? 0 : v / r.down + 1);
    }
    E1[s] = e;
    n_out[s] = (int32_t)(e - E0);
    rows[s] = RsRow{P0 - rs->K, std::max(0LL, P0 - rs->K), P1, E0, e - E0, e - E0};
    max_out = std::max(max_out, e - E0);
  }

  // ---- device: one table copy, prep, resample ----
  rc = rs->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  rc = rs_launch(ctx, r, rs->taps, rs->win, rs->cap, rs->cap, nullptr, rs->d_rows<0>(), S, 0, max_out, y_dev, rs->out_pitch, st);
  if (rc) return rc;
  rs->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_resample_stream_push_host(vtts_ctx* ctx, vtts_resample_stream* rs, const float* x, const int32_t* n_new, const uint8_t* flags,
                                   float* y, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "resample_stream_push_host", rs, x && y);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)rs->S * rs->F * 4), o_y = hs.out((size_t)rs->S * rs->out_pitch * 4, y);
  return hs.run([&](cudaStream_t st) {
    return vtts_resample_stream_push(ctx, rs, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, st);
  });
}
