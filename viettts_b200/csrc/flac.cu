// FLAC encoding of synthesized audio: a native, mono, 16-bit FLAC stream per row, in the streamable subset (RFC 9639).
// oracle/flac_oracle.py is the definition; the device writes its bytes exactly, in every vtts_precision mode, because
// every decision is made in integers or in correctly rounded fp64 (__dadd_rn / __dmul_rn / __ddiv_rn, never an FMA).
//
// A row of n samples (PCM-16 codes of the float input, VTTS_PCM16_OF) gives ceil(n / block) frames after the 42-byte
// stream header.  Three launches:
//   analysis  grid (frames, B), 256 threads: one CTA per frame loads and quantizes its block, tests for CONSTANT, takes
//             the integer autocorrelation of the windowed block (int32 products, int64 sums), runs Levinson-Durbin and
//             the coefficient quantization of orders 1..12 in one thread, then for each of the 17 predictors (FIXED
//             0..4, LPC 1..12) sums u >> k (u the zigzag residual, k = 0..14) per finest Rice partition in registers,
//             merges the partitions level by level in shared memory and keeps the exact cheapest candidate
//             (VERBATIM last).  It writes a small per-frame descriptor with the frame's byte size.
//   offsets   grid B, 1024 threads: a per-row exclusive scan of the frame sizes after the stream header, the row's
//             byte count, and the stream header itself (STREAMINFO with the min / max frame size).
//   pack      grid (frames, B), 256 threads: recomputes the chosen residual and its Rice parameters, takes a
//             block-wide scan of the per-sample code lengths for their bit offsets, writes the frame MSB-first into a
//             shared-memory bit buffer with its header and CRC-8, computes the CRC-16 split over the threads (the CRC is
//             linear: each thread's segment CRC is carried past the bytes after it by a power of x mod the polynomial
//             and the parts are XORed) and copies the frame to its offset.
#include <climits>

#include "pcm16.cuh"
#include "stream_common.cuh"

namespace {

constexpr int T = 256;            // threads of a frame CTA
constexpr int MAXB = 4096;        // largest block
constexpr int NK = 15;            // Rice parameters 0..14
constexpr int MAXP = 8;           // largest partition order
constexpr int NPART = 1 << MAXP;
constexpr int MAXO = 12;          // largest LPC order
constexpr int HDR = 42;           // "fLaC" + STREAMINFO
constexpr int FRAME_HDR_MAX = 15; // 4 + 6 (frame number) + 2 (block size) + 2 (rate) + 1 (CRC-8)
constexpr int MAX_FRAME = FRAME_HDR_MAX + 1 + 2 * MAXB + 2;
constexpr int SCAN_T = 1024;      // threads of the offsets CTA

enum { SUB_CONST = 0, SUB_VERB = 1, SUB_FIXED = 2, SUB_LPC = 3 };

struct FrameDesc {
  long long off;        // byte offset of the frame in its row (offsets kernel)
  int bytes;            // frame size, 0 for a frame past the row's end
  int type, order, porder, shift, precision;
  int q[MAXO];
};

struct RateCode {
  int code, extra_bytes, extra;
};

bool block_ok(int block) { return block == 256 || block == 512 || block == 1024 || block == 2048 || block == 4096; }

// the frame header's rate field (flac_oracle.rate_code); false for a rate FLAC cannot state
bool rate_code(int rate, RateCode* rc) {
  static const int table[][2] = {{88200, 1}, {176400, 2}, {192000, 3}, {8000, 4},  {16000, 5}, {22050, 6},
                                 {24000, 7}, {32000, 8},  {44100, 9},  {48000, 10}, {96000, 11}};
  if (rate < 1) return false;
  for (const auto& t : table)
    if (t[0] == rate) return *rc = {t[1], 0, 0}, true;
  if (rate % 1000 == 0 && rate / 1000 <= 255) return *rc = {12, 1, rate / 1000}, true;
  if (rate <= 65535) return *rc = {13, 2, rate}, true;
  if (rate % 10 == 0 && rate / 10 <= 65535) return *rc = {14, 2, rate / 10}, true;
  return false;
}

__host__ __device__ int utf8_len(long long v) {
  return v < 0x80 ? 1 : v < 0x800 ? 2 : v < 0x10000 ? 3 : v < 0x200000 ? 4 : v < 0x4000000 ? 5 : v < 0x80000000LL ? 6 : 7;
}

__device__ int header_bytes(int n, int block, long long number, const RateCode& rc) {
  return 4 + utf8_len(number) + (n == block ? 0 : (n <= 256 ? 1 : 2)) + rc.extra_bytes + 1;
}

__device__ int block_code(int block) { return 31 - __clz(block); }   // 256 -> 8 .. 4096 -> 12

__device__ int precision_of(int n) {
  return n <= 192 ? 7 : n <= 384 ? 8 : n <= 576 ? 9 : n <= 1152 ? 10 : n <= 2304 ? 11 : 12;
}

// the largest partition order p <= 8 with n divisible by 2^p and (n >> p) > order
__device__ int max_porder(int n, int order) {
  int p = 0;
  while (p < MAXP && n % (2 << p) == 0 && (n >> (p + 1)) > order) ++p;
  return p;
}

// Q15 window: a smoothstep taper over L = n >> 2 samples at each end (flac_oracle.window)
__device__ int window_q15(int i, int n) {
  const int L = n >> 2;
  if (i >= L && i < n - L) return 32768;
  const long long a = 2 * (long long)(i < L ? i : n - 1 - i) + 1, D = 2 * (long long)L;
  return (int)((32768 * (3 * a * a * D - 2 * a * a * a)) / (D * D * D));
}

// block-wide sums of v[0..N) (every thread gets them); tmp holds (T / 32) * N values
template <int N, class V>
__device__ void block_sum(V* v, V* tmp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int i = 0; i < N; ++i)
    for (int o = 16; o; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
  if (lane == 0)
    for (int i = 0; i < N; ++i) tmp[warp * N + i] = v[i];
  __syncthreads();
  for (int i = 0; i < N; ++i) {
    V s = 0;
    for (int w = 0; w < nw; ++w) s += tmp[w * N + i];
    v[i] = s;
  }
  __syncthreads();
}

// block-wide exclusive prefix sum of v; tmp holds 32 values; `total` gets the sum
template <class V>
__device__ V block_scan(V v, V* tmp, V* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  V x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const V y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) tmp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    V w = lane < nw ? tmp[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const V y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < nw) tmp[lane] = w;
  }
  __syncthreads();
  const V before = (warp ? tmp[warp - 1] : 0) + x - v;
  *total = tmp[nw - 1];
  __syncthreads();
  return before;
}

struct Cand {
  int type, order, shift;
  const int* q;
};

// residual of candidate c at sample t >= order, in int64
__device__ __forceinline__ long long residual(const int* x, int t, const Cand& c) {
  if (c.type == SUB_FIXED) {
    switch (c.order) {
      case 0: return x[t];
      case 1: return (long long)x[t] - x[t - 1];
      case 2: return (long long)x[t] - 2LL * x[t - 1] + x[t - 2];
      case 3: return (long long)x[t] - 3LL * x[t - 1] + 3LL * x[t - 2] - x[t - 3];
      default: return (long long)x[t] - 4LL * x[t - 1] + 6LL * x[t - 2] - 4LL * x[t - 3] + x[t - 4];
    }
  }
  long long s = 0;
  for (int j = 0; j < c.order; ++j) s += (long long)(c.q[j] * x[t - 1 - j]);
  return x[t] - (s >> c.shift);
}

__device__ __forceinline__ unsigned zigzag(long long r) { return (unsigned)(r >= 0 ? 2 * r : -2 * r - 1); }

struct AnaSmem {
  int x[MAXB];
  union {
    int xw[MAXB];
    unsigned long long sums[NPART * NK];   // [partition][k] at the current level
  };
  unsigned long long wacc[(T / 32) * NK];
  long long red[(T / 32) * (MAXO + 1)];
  long long R[MAXO + 1];
  long long tot[MAXP + 1];
  int qlp[MAXO][MAXO], qshift[MAXO], qok[MAXO];
  int best_bits, best_type, best_order, best_p;
};

// s.sums[j][k] = sum over finest partition j (order pf) of u >> k, samples t >= order; false (block-uniform) when a
// residual leaves the int32 range
__device__ bool part_sums(AnaSmem& s, int n, int pf, const Cand& c) {
  const int nparts = 1 << pf, m = n >> pf, tpp = T / nparts;   // threads per partition
  const int part = threadIdx.x / tpp, sub = threadIdx.x % tpp, per = (m + tpp - 1) / tpp;
  const int lo = part * m + min(sub * per, m), hi = part * m + min((sub + 1) * per, m);
  unsigned long long acc[NK];
#pragma unroll
  for (int k = 0; k < NK; ++k) acc[k] = 0;
  int bad = 0;
  for (int t = max(lo, c.order); t < hi; ++t) {
    const long long r = residual(s.x, t, c);
    bad |= r < INT_MIN || r > INT_MAX;
    const unsigned u = zigzag(r);
#pragma unroll
    for (int k = 0; k < NK; ++k) acc[k] += u >> k;
  }
  const int w = min(tpp, 32);
#pragma unroll
  for (int k = 0; k < NK; ++k)
    for (int o = 1; o < w; o <<= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  if (tpp <= 32) {
    if (sub == 0)
      for (int k = 0; k < NK; ++k) s.sums[part * NK + k] = acc[k];
  } else if ((threadIdx.x & 31) == 0) {
    for (int k = 0; k < NK; ++k) s.wacc[(threadIdx.x >> 5) * NK + k] = acc[k];
  }
  __syncthreads();
  if (tpp > 32)
    for (int i = threadIdx.x; i < nparts * NK; i += T) {
      const int j = i / NK, k = i % NK, wpp = tpp / 32;
      unsigned long long v = 0;
      for (int q = 0; q < wpp; ++q) v += s.wacc[(j * wpp + q) * NK + k];
      s.sums[i] = v;
    }
  return !__syncthreads_or(bad);
}

// cheapest k (the smaller on a tie) and its bits for a partition of cnt residuals
__device__ __forceinline__ int rice_k(const unsigned long long* sk, long long cnt, long long* bits) {
  long long b = (long long)sk[0] + cnt;
  int kb = 0;
  for (int k = 1; k < NK; ++k) {
    const long long v = (long long)sk[k] + cnt * (k + 1);
    if (v < b) b = v, kb = k;
  }
  *bits = b;
  return kb;
}

// merges level p of s.sums into level p - 1 in place
__device__ void merge_level(AnaSmem& s, int p) {
  const int items = (1 << (p - 1)) * NK;
  unsigned long long v[(NPART / 2 * NK + T - 1) / T];
#pragma unroll
  for (int i = 0; i < (int)(sizeof(v) / sizeof(v[0])); ++i) {
    const int idx = threadIdx.x + i * T;
    if (idx < items) v[i] = s.sums[(idx / NK) * 2 * NK + idx % NK] + s.sums[((idx / NK) * 2 + 1) * NK + idx % NK];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < (int)(sizeof(v) / sizeof(v[0])); ++i) {
    const int idx = threadIdx.x + i * T;
    if (idx < items) s.sums[idx] = v[i];
  }
  __syncthreads();
}

// Rice bits of the residual section (2 + 4 + partitions) of candidate c at its best partition order; -1 if skipped
__device__ long long rice_cost(AnaSmem& s, int n, int pf, const Cand& c, int* best_p) {
  if (threadIdx.x <= MAXP) s.tot[threadIdx.x] = 0;
  if (!part_sums(s, n, pf, c)) return -1;   // its barriers order the tot reset before the sums below
  const int pmax = max_porder(n, c.order);
  for (int p = pf; p >= 0; --p) {
    if (p <= pmax) {
      long long part = 0;
      for (int j = threadIdx.x; j < (1 << p); j += T) {
        long long b;
        rice_k(&s.sums[j * NK], (n >> p) - (j == 0 ? c.order : 0), &b);
        part += 4 + b;
      }
      for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      if ((threadIdx.x & 31) == 0 && part) atomicAdd((unsigned long long*)&s.tot[p], (unsigned long long)part);
    }
    if (p) merge_level(s, p);
  }
  __syncthreads();
  long long best = -1;
  for (int p = 0; p <= pmax; ++p)
    if (best < 0 || 6 + s.tot[p] < best) best = 6 + s.tot[p], *best_p = p;
  __syncthreads();
  return best;
}

// Levinson-Durbin over R[0..12] and libFLAC's coefficient quantization at precision P, for the orders < n (one thread)
__device__ void lpc_analysis(AnaSmem& s, int n, int P) {
  for (int o = 0; o < MAXO; ++o) s.qok[o] = 0;
  double a[MAXO], na[MAXO];
  double err = (double)s.R[0];
  for (int i = 1; i <= MAXO; ++i) {
    if (!(err > 0.0)) break;
    double acc = (double)s.R[i];
    for (int j = 0; j < i - 1; ++j) acc = __dadd_rn(acc, -__dmul_rn(a[j], (double)s.R[i - 1 - j]));
    const double k = __ddiv_rn(acc, err);
    for (int j = 0; j < i - 1; ++j) na[j] = __dadd_rn(a[j], -__dmul_rn(k, a[i - 2 - j]));
    na[i - 1] = k;
    err = __dmul_rn(err, __dadd_rn(1.0, -__dmul_rn(k, k)));
    bool fin = true;
    double cmax = 0.0;
    for (int j = 0; j < i; ++j) {
      a[j] = na[j];
      fin &= isfinite(a[j]);
      cmax = fmax(cmax, fabs(a[j]));
    }
    if (!fin) break;
    if (i >= n || !(cmax > 0.0)) continue;
    int e;
    frexp(cmax, &e);
    const int shift = min(max(P - e, 0), 15);
    const double scale = (double)(1 << shift), qmax = (double)((1 << (P - 1)) - 1), qmin = -(double)(1 << (P - 1));
    double ef = 0.0;
    for (int j = 0; j < i; ++j) {
      ef = __dadd_rn(ef, __dmul_rn(a[j], scale));
      const double q = fmin(fmax(rint(ef), qmin), qmax);
      ef = __dadd_rn(ef, -q);
      s.qlp[i - 1][j] = (int)q;
    }
    s.qshift[i - 1] = shift;
    s.qok[i - 1] = 1;
  }
}

// What one launch encodes of row b: sample t of the row is a[t] for t < na, else c[t - na] (a stream slot's carried
// samples, then its push's new ones); frames [0, nfr) cover samples [0, n), frame f is frame number frame0 + f; with
// head the row's bytes start with the stream header (total samples `total`, the min / max frame size when minmax).
struct FlacRow {
  const float* a;
  const float* c;
  int na, n, nfr, head, minmax;
  long long frame0, total;
};

// per row, from the offsets and place kernels: the row's bytes, its min / max frame size and where it starts in y
struct RowOut {
  long long bytes, start;
  int fmin, fmax;
};

struct FlacArgs {
  const FlacRow* rows;  // [B]
  int B, block;
  RateCode rc;
  int rate;
  int nf;               // frame slots per row
  FrameDesc* desc;      // [B][nf]
  RowOut* ro;           // [B]
  uint8_t* y;
  long long pitch;      // > 0: row b starts at b * pitch (one-shot); 0: the rows are packed one after another (stream)
  int* nbytes;          // one-shot: [B] row byte counts
  int* tbl;             // stream: [B][2] (offset, count) of each row in y
};

__device__ __forceinline__ float row_sample(const FlacRow& r, long long t) { return t < r.na ? r.a[t] : r.c[t - r.na]; }

// the one-shot rows: row b of x [B][S] holds n_in[b] samples (S without n_in)
__global__ void flac_rows_oneshot(const float* x, const int* n_in, int S, int B, int block, FlacRow* rows) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int n = n_in ? min(max(n_in[b], 0), S) : S;
  rows[b] = FlacRow{x + (size_t)b * S, nullptr, n, n, (int)((n + (long long)block - 1) / block), 1, 1, 0, n};
}

__global__ void __launch_bounds__(T) flac_analyze(FlacArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AnaSmem& s = *reinterpret_cast<AnaSmem*>(smem_raw);
  const int b = blockIdx.y, f = blockIdx.x;
  const FlacRow r = A.rows[b];
  FrameDesc& d = A.desc[(size_t)b * A.nf + f];
  const long long t0 = (long long)f * A.block;
  if (f >= r.nfr) {
    if (threadIdx.x == 0) d.bytes = 0;
    return;
  }
  const int n = (int)min((long long)A.block, r.n - t0);
  int diff = 0;
  for (int t = threadIdx.x; t < n; t += T) s.x[t] = VTTS_PCM16_OF(row_sample(r, t0 + t));
  __syncthreads();
  for (int t = threadIdx.x; t < n; t += T) diff |= s.x[t] != s.x[0];
  const int hb = header_bytes(n, A.block, r.frame0 + f, A.rc);
  if (!__syncthreads_or(diff)) {
    if (threadIdx.x == 0) d.type = SUB_CONST, d.bytes = hb + 3 + 2;
    return;
  }
  // windowed autocorrelation, lags 0..12
  for (int t = threadIdx.x; t < n; t += T) s.xw[t] = (s.x[t] * window_q15(t, n) + (1 << 14)) >> 15;
  __syncthreads();
  long long R[MAXO + 1];
#pragma unroll
  for (int l = 0; l <= MAXO; ++l) R[l] = 0;
  for (int t = threadIdx.x; t < n; t += T) {
    const int v = s.xw[t];
#pragma unroll
    for (int l = 0; l <= MAXO; ++l)
      if (t >= l) R[l] += (long long)(v * s.xw[t - l]);
  }
  block_sum<MAXO + 1>(R, s.red);
  const int P = precision_of(n);
  if (threadIdx.x == 0) {
    for (int l = 0; l <= MAXO; ++l) s.R[l] = R[l];
    lpc_analysis(s, n, P);
    s.best_bits = 8 + 16 * n;   // VERBATIM, which wins only where no predictor is cheaper (it is compared last)
    s.best_type = -1;
  }
  __syncthreads();
  const int pf = max_porder(n, 0);
  for (int ci = 0; ci < 5 + MAXO; ++ci) {
    Cand c;
    int sub_fixed;
    if (ci < 5) {
      c = {SUB_FIXED, ci, 0, nullptr};
      sub_fixed = 8 + 16 * ci;
    } else {
      const int o = ci - 4;
      if (!s.qok[o - 1]) continue;
      c = {SUB_LPC, o, s.qshift[o - 1], s.qlp[o - 1]};
      sub_fixed = 8 + 16 * o + 4 + 5 + P * o;
    }
    if (c.order >= n) continue;
    int p = 0;
    const long long rb = rice_cost(s, n, pf, c, &p);
    if (threadIdx.x == 0 && rb >= 0) {
      const long long bits = sub_fixed + rb;
      // candidates come in the order of the definition: a later one must be strictly cheaper; VERBATIM (the initial
      // best) is last, so a predictor that only ties it wins
      if (bits < s.best_bits || (s.best_type < 0 && bits == s.best_bits))
        s.best_bits = (int)bits, s.best_type = c.type, s.best_order = c.order, s.best_p = p;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int type = s.best_type < 0 ? SUB_VERB : s.best_type;
    d.type = type;
    d.order = s.best_order;
    d.porder = s.best_p;
    d.precision = P;
    if (type == SUB_LPC) {
      d.shift = s.qshift[s.best_order - 1];
      for (int j = 0; j < s.best_order; ++j) d.q[j] = s.qlp[s.best_order - 1][j];
    }
    d.bytes = hb + (s.best_bits + 7) / 8 + 2;
  }
}

// per row: frame offsets after the stream header (when the row has one), the row's byte count and min / max frame
__global__ void __launch_bounds__(SCAN_T) flac_offsets(FlacArgs A) {
  __shared__ long long tmp[32];
  __shared__ int mn, mx;
  const int b = blockIdx.x;
  const FlacRow r = A.rows[b];
  FrameDesc* d = A.desc + (size_t)b * A.nf;
  long long carry = r.head ? HDR : 0;
  int lmin = INT_MAX, lmax = 0;
  for (int f0 = 0; f0 < r.nfr; f0 += SCAN_T) {
    const int f = f0 + threadIdx.x;
    const long long v = f < r.nfr ? d[f].bytes : 0;
    long long total;
    const long long ex = block_scan<long long>(v, tmp, &total);
    if (f < r.nfr) {
      d[f].off = carry + ex;
      lmin = min(lmin, (int)v);
      lmax = max(lmax, (int)v);
    }
    carry += total;
  }
  for (int o = 16; o; o >>= 1) {
    lmin = min(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
    lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  }
  if (threadIdx.x == 0) mn = INT_MAX, mx = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicMin(&mn, lmin), atomicMax(&mx, lmax);
  __syncthreads();
  if (threadIdx.x == 0) A.ro[b] = RowOut{carry, 0, r.nfr ? mn : 0, r.nfr ? mx : 0};
}

// one CTA: where each row starts (b * pitch, or packed after the rows before it), the row byte counts or the (offset,
// count) table, and the stream header of every row that has one
__global__ void __launch_bounds__(SCAN_T) flac_place(FlacArgs A) {
  __shared__ long long tmp[32];
  long long carry = 0;
  for (int b0 = 0; b0 < A.B; b0 += SCAN_T) {
    const int b = b0 + threadIdx.x;
    const long long v = b < A.B ? A.ro[b].bytes : 0;
    long long total;
    const long long ex = block_scan<long long>(v, tmp, &total);
    if (b < A.B) {
      const long long start = A.pitch ? b * A.pitch : carry + ex;
      A.ro[b].start = start;
      if (A.nbytes) A.nbytes[b] = (int)v;
      if (A.tbl) A.tbl[2 * b] = (int)start, A.tbl[2 * b + 1] = (int)v;
      const FlacRow r = A.rows[b];
      if (r.head) {
        uint8_t* y = A.y + start;
        const unsigned long long fmin = r.minmax ? A.ro[b].fmin : 0, fmax = r.minmax ? A.ro[b].fmax : 0, blk = A.block;
        const unsigned long long n = r.total;
        const uint8_t h[8] = {'f', 'L', 'a', 'C', 0x80, 0, 0, 34};
        for (int i = 0; i < 8; ++i) y[i] = h[i];
        // STREAMINFO: min / max block (16 + 16), min / max frame (24 + 24), rate (20), channels - 1 (3), bits - 1 (5),
        // total samples (36), MD5 (128, zero: unknown)
        const unsigned long long v0 = blk << 48 | blk << 32 | fmin << 8 | fmax >> 16;
        const unsigned long long v1 = (fmax & 0xFFFF) << 48 | (unsigned long long)A.rate << 28 | 0ull << 25 | 15ull << 20 |
                                      (n >> 16 & 0xFFFFF);
        for (int i = 0; i < 8; ++i) y[8 + i] = (uint8_t)(v0 >> (56 - 8 * i));
        for (int i = 0; i < 8; ++i) y[16 + i] = (uint8_t)(v1 >> (56 - 8 * i));
        y[24] = (uint8_t)(n >> 8);
        y[25] = (uint8_t)n;
        for (int i = 26; i < HDR; ++i) y[i] = 0;
      }
    }
    carry += total;
  }
}

__device__ __forceinline__ void put_bits(unsigned* buf, long long pos, unsigned v, int w) {
  const int sh = (int)(pos & 31);
  unsigned* p = buf + (pos >> 5);
  if (sh + w <= 32) {
    atomicOr(p, v << (32 - sh - w));
  } else {
    atomicOr(p, v >> (sh + w - 32));
    atomicOr(p + 1, v << (64 - sh - w));
  }
}

__device__ __forceinline__ unsigned get_byte(const unsigned* buf, int i) { return (buf[i >> 2] >> (24 - 8 * (i & 3))) & 0xFF; }

// a(x) b(x) mod x^16 + x^15 + x^2 + 1
__device__ unsigned gf16_mul(unsigned a, unsigned b) {
  unsigned r = 0;
  for (int i = 15; i >= 0; --i) {
    r = (r << 1) ^ (r & 0x8000 ? 0x8005 : 0);
    r &= 0xFFFF;
    if (b >> i & 1) r ^= a;
  }
  return r;
}

// x^(8 z) mod the CRC-16 polynomial: the factor that carries a CRC past z zero bytes
__device__ unsigned gf16_xpow8(int z) {
  unsigned r = 1, base = 0x100;
  while (z) {
    if (z & 1) r = gf16_mul(r, base);
    base = gf16_mul(base, base);
    z >>= 1;
  }
  return r;
}

// the analysis layout (part_sums runs on it again), then the packing's own fields; the frame's bit buffer takes the
// place of the partition sums once the Rice parameters are known
struct PackSmem {
  AnaSmem a;
  int q[MAXO];
  unsigned char kk[NPART];
  int tmp[32];
  unsigned crc[T / 32];
};
constexpr int BUF_WORDS = (MAX_FRAME + 3) / 4 + 1;
static_assert(BUF_WORDS * 4 <= NPART * NK * 8, "the bit buffer fits in the partition sums");

__global__ void __launch_bounds__(T) flac_pack(FlacArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PackSmem& s = *reinterpret_cast<PackSmem*>(smem_raw);
  AnaSmem& as = s.a;
  unsigned* const buf = reinterpret_cast<unsigned*>(as.sums);
  const int b = blockIdx.y, f = blockIdx.x;
  const FlacRow r = A.rows[b];
  if (f >= r.nfr) return;
  const long long t0 = (long long)f * A.block, number = r.frame0 + f;
  const FrameDesc d = A.desc[(size_t)b * A.nf + f];
  const int n = (int)min((long long)A.block, r.n - t0);
  for (int t = threadIdx.x; t < n; t += T) as.x[t] = VTTS_PCM16_OF(row_sample(r, t0 + t));
  if (threadIdx.x < MAXO) s.q[threadIdx.x] = d.q[threadIdx.x];
  __syncthreads();
  const Cand c = {d.type, d.order, d.shift, s.q};
  const int p = d.porder, m = n >> p;
  if (d.type == SUB_FIXED || d.type == SUB_LPC) {
    // the Rice parameter of each partition at the chosen order, as the analysis found it
    const int pf = max_porder(n, 0);
    part_sums(as, n, pf, c);
    for (int q = pf; q > p; --q) merge_level(as, q);
    for (int j = threadIdx.x; j < (1 << p); j += T) {
      long long bits;
      s.kk[j] = (unsigned char)rice_k(&as.sums[j * NK], m - (j == 0 ? c.order : 0), &bits);
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < BUF_WORDS; i += T) buf[i] = 0;
  __syncthreads();
  const int hb = header_bytes(n, A.block, number, A.rc);
  const long long sub0 = 8LL * hb;
  // per-sample code lengths: each thread owns a contiguous run of samples
  const int per = (n + T - 1) / T, lo = min((int)threadIdx.x * per, n), hi = min(lo + per, n);
  if (d.type == SUB_VERB) {
    for (int t = lo; t < hi; ++t) put_bits(buf, sub0 + 8 + 16LL * t, (unsigned)as.x[t] & 0xFFFF, 16);
  } else if (d.type != SUB_CONST) {
    int len = 0;
    for (int t = max(lo, c.order); t < hi; ++t) {
      const int k = s.kk[t / m];
      len += (int)(zigzag(residual(as.x, t, c)) >> k) + 1 + k;
    }
    int total;
    const int before = block_scan<int>(len, s.tmp, &total);
    const long long res0 = sub0 + 8 + 16LL * c.order + (d.type == SUB_LPC ? 9 + d.precision * c.order : 0) + 6;
    // partition j's 4-bit parameter precedes its first code; codes before sample t: before + the ones of this thread
    long long at = before;
    for (int t = max(lo, c.order); t < hi; ++t) {
      const int j = t / m, k = s.kk[j];
      const bool first = t == (j == 0 ? c.order : j * m);
      const long long base = res0 + 4LL * (j + 1) + at;
      if (first) put_bits(buf, base - 4, k, 4);
      const unsigned u = zigzag(residual(as.x, t, c));
      const int q = (int)(u >> k);
      put_bits(buf, base + q, (1u << k) | (u & ((1u << k) - 1)), k + 1);
      at += q + 1 + k;
    }
  }
  if (threadIdx.x == 0) {
    // frame header and its CRC-8
    uint8_t h[FRAME_HDR_MAX];
    int i = 0;
    h[i++] = 0xFF;
    h[i++] = 0xF8;
    const int bc = n == A.block ? block_code(A.block) : (n <= 256 ? 6 : 7);
    h[i++] = (uint8_t)(bc << 4 | A.rc.code);
    h[i++] = 0x08;
    const int ul = utf8_len(number);
    if (ul == 1) {
      h[i++] = (uint8_t)number;
    } else {
      h[i++] = (uint8_t)(((0xFF00 >> ul) & 0xFF) | (number >> (6 * (ul - 1))));
      for (int k = ul - 2; k >= 0; --k) h[i++] = (uint8_t)(0x80 | ((number >> (6 * k)) & 0x3F));
    }
    if (bc == 6) h[i++] = (uint8_t)(n - 1);
    if (bc == 7) h[i++] = (uint8_t)((n - 1) >> 8), h[i++] = (uint8_t)(n - 1);
    if (A.rc.extra_bytes == 2) h[i++] = (uint8_t)(A.rc.extra >> 8);
    if (A.rc.extra_bytes) h[i++] = (uint8_t)A.rc.extra;
    unsigned c8 = 0;
    for (int k = 0; k < i; ++k) {
      c8 ^= h[k];
      for (int r = 0; r < 8; ++r) c8 = (c8 & 0x80 ? (c8 << 1) ^ 0x07 : c8 << 1) & 0xFF;
    }
    h[i++] = (uint8_t)c8;
    for (int k = 0; k < i; ++k) put_bits(buf, 8LL * k, h[k], 8);
    // subframe header and its fixed fields
    long long q = sub0;
    const int tcode = d.type == SUB_CONST ? 0 : d.type == SUB_VERB ? 1 : d.type == SUB_FIXED ? (0x08 | c.order) : (0x20 | (c.order - 1));
    put_bits(buf, q, tcode << 1, 8);
    q += 8;
    if (d.type == SUB_CONST) put_bits(buf, q, (unsigned)as.x[0] & 0xFFFF, 16);
    if (d.type == SUB_FIXED || d.type == SUB_LPC) {
      for (int j = 0; j < c.order; ++j, q += 16) put_bits(buf, q, (unsigned)as.x[j] & 0xFFFF, 16);
      if (d.type == SUB_LPC) {
        put_bits(buf, q, d.precision - 1, 4);
        put_bits(buf, q + 4, d.shift, 5);
        q += 9;
        for (int j = 0; j < c.order; ++j, q += d.precision) put_bits(buf, q, (unsigned)d.q[j] & ((1u << d.precision) - 1), d.precision);
      }
      put_bits(buf, q, p, 6);   // method 0 (2 bits), partition order (4 bits)
    }
  }
  __syncthreads();
  // CRC-16 of bytes [0, L), split over the threads and carried past the bytes after each segment
  const int L = d.bytes - 2, seg = (L + T - 1) / T, a = min((int)threadIdx.x * seg, L), e = min(a + seg, L);
  unsigned crc = 0;
  for (int i = a; i < e; ++i) {
    crc ^= get_byte(buf, i) << 8;
    for (int r = 0; r < 8; ++r) crc = (crc & 0x8000 ? (crc << 1) ^ 0x8005 : crc << 1) & 0xFFFF;
  }
  if (e > a && L - e > 0) crc = gf16_mul(crc, gf16_xpow8(L - e));
  for (int o = 16; o; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
  if ((threadIdx.x & 31) == 0) s.crc[threadIdx.x >> 5] = crc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned c16 = 0;
    for (int w = 0; w < T / 32; ++w) c16 ^= s.crc[w];
    put_bits(buf, 8LL * L, c16, 16);
  }
  __syncthreads();
  uint8_t* yo = A.y + A.ro[b].start + d.off;
  for (int i = threadIdx.x; i < d.bytes; i += T) yo[i] = (uint8_t)get_byte(buf, i);
}

long long flac_bound(long long S, int block) {
  const long long nf = (S + block - 1) / block;
  return HDR + nf * (FRAME_HDR_MAX + 1 + 2) + 2 * S;
}

bool overlaps(const void* a, size_t an, const void* b, size_t bn) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + bn && y < x + an;
}

// the block, rate and batch shape of a one-shot call of entry point `who` (an empty row is a valid stream), and the
// bytes a row can take
int flac_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, int block, RateCode* rc, long long* bound) {
  if (!block_ok(block)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: block %d (256, 512, 1024, 2048 or 4096)", who, block);
  if (!rate_code(rate, rc))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: rate %d has no FLAC frame-header code (a table rate, kHz <= 255, Hz <= 65535 or "
                     "tens of Hz <= 655350)", who, rate);
  const int r = batch_check(ctx, who, B, S, S_ANY, 0);
  if (r) return r;
  *bound = flac_bound(S, block);
  if (*bound > INT_MAX) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: S=%d: a row's bound of %lld bytes exceeds 2^31 - 1", who, S, *bound);
  return VTTS_OK;
}

// the device buffers of a one-shot call: y rows `pitch` bytes apart, each at least the bound, all three apart
int flac_buffers(vtts_ctx* ctx, const char* who, const void* x, const void* y, const void* nb, int B, int S, long long pitch, long long bound) {
  if (pitch < bound) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: y_pitch %lld below the bound %lld (vtts_flac_bound)", who, pitch, bound);
  if ((S && !x) || !y || !nb) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
  const size_t xb = (size_t)B * S * 4, yb = (size_t)(B - 1) * pitch + bound, nbb = (size_t)B * 4;
  if ((S && (overlaps(x, xb, y, yb) || overlaps(x, xb, nb, nbb))) || overlaps(y, yb, nb, nbb))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: the buffers overlap", who);
  return VTTS_OK;
}

// the analysis and packing CTAs take a little over the 48 KB of shared memory a launch gets without asking; set once
// per device
int flac_smem_setup(vtts_ctx* ctx) {
  static unsigned long long done = 0;
  const unsigned long long bit = 1ull << (ctx->device & 63);
  if (done & bit) return VTTS_OK;
  VTTS_CUDA(cudaFuncSetAttribute(flac_analyze, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(AnaSmem)));
  VTTS_CUDA(cudaFuncSetAttribute(flac_pack, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PackSmem)));
  done |= bit;
  return VTTS_OK;
}

// analysis, offsets, placement and packing of the rows in A.rows (on the device); A.nf frame slots per row
int flac_launch(vtts_ctx* ctx, const FlacArgs& A, cudaStream_t st) {
  int r = flac_smem_setup(ctx);
  if (r) return r;
  if (A.nf) flac_analyze<<<dim3(A.nf, A.B), T, sizeof(AnaSmem), st>>>(A);
  flac_offsets<<<A.B, SCAN_T, 0, st>>>(A);
  flac_place<<<1, SCAN_T, 0, st>>>(A);
  if (A.nf) flac_pack<<<dim3(A.nf, A.B), T, sizeof(PackSmem), st>>>(A);
  ctx->launches += A.nf ? 4 : 2;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// a stream slot's samples [from, from + cnt) of the push (carried, then new) become its carried samples
__global__ void flac_carry(const FlacRow* rows, const int* keep, int block, float* dst) {
  const int s = blockIdx.x, cnt = keep[2 * s + 1];
  const FlacRow r = rows[s];
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) dst[(size_t)s * block + i] = row_sample(r, (long long)keep[2 * s] + i);
}

}  // namespace

int64_t vtts_flac_bound(int S, int block) {
  if (S < 0 || !block_ok(block)) return -1;
  return flac_bound(S, block);
}

int vtts_flac_rate_code(int rate) {
  RateCode rc;
  return rate_code(rate, &rc) ? rc.code : -1;
}

namespace {

int flac_oneshot(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, int block, const RateCode& rc, uint8_t* y,
                 int64_t y_pitch, int32_t* nbytes, cudaStream_t st) {
  const int nf = (S + block - 1) / block;
  const auto carve = [&](Arena& a, FrameDesc** d, FlacRow** rows, RowOut** ro) {
    *d = a.take<FrameDesc>((size_t)B * nf);
    *rows = a.take<FlacRow>(B);
    *ro = a.take<RowOut>(B);
  };
  FrameDesc* d;
  FlacRow* rows;
  RowOut* ro;
  Arena m(nullptr, 0, true);
  carve(m, &d, &rows, &ro);
  if (const int r = ctx->ensure_ws(m.off)) return r;
  Arena a(ctx->ws, ctx->ws_bytes, false);
  carve(a, &d, &rows, &ro);
  flac_rows_oneshot<<<(B + 255) / 256, 256, 0, st>>>(x, n_in, S, B, block, rows);
  ctx->launches++;
  const FlacArgs A{rows, B, block, rc, rate, nf, d, ro, y, y_pitch, nbytes, nullptr};
  return flac_launch(ctx, A, st);
}

}  // namespace

int vtts_flac_encode(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, int block, uint8_t* y_dev,
                     int64_t y_pitch, int32_t* nbytes_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  RateCode rc;
  long long bound;
  int r = flac_args(ctx, "flac_encode", B, S, rate, block, &rc, &bound);
  if (!r) r = flac_buffers(ctx, "flac_encode", x_dev, y_dev, nbytes_dev, B, S, y_pitch, bound);
  if (r) return r;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return flac_oneshot(ctx, x_dev, n_dev, B, S, rate, block, rc, y_dev, y_pitch, nbytes_dev, (cudaStream_t)stream);
}

// two fetches: each row's byte count, then as many bytes of every row as the longest one took
int vtts_flac_encode_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, int block, uint8_t* y,
                          int64_t y_pitch, int32_t* nbytes) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  RateCode rc;
  long long pitch;
  int r = flac_args(ctx, "flac_encode_host", B, S, rate, block, &rc, &pitch);
  if (r) return r;
  HostStage hs(ctx);
  r = flac_buffers(ctx, "flac_encode_host", x, y, nbytes, B, S, y_pitch, pitch);
  if (!r) r = hs.rows("flac_encode_host", x, n_in, B, S);
  if (r) return r;
  const size_t o_y = hs.out((size_t)B * pitch), o_nb = hs.out((size_t)B * 4, nbytes);
  r = hs.run([&](cudaStream_t st) {
    return flac_oneshot(ctx, hs.x(), hs.n(), B, S, rate, block, rc, hs.dev<uint8_t>(o_y), pitch, hs.dev<int32_t>(o_nb), st);
  });
  if (r) return r;
  // then one copy of the longest row's bytes from every row, and each row's own bytes out of it
  int width = 0;
  for (int b = 0; b < B; ++b) width = std::max(width, (int)nbytes[b]);
  char* hp = (char*)ctx->hpin + o_y;
  VTTS_CUDA(cudaMemcpy2DAsync(hp, pitch, hs.dev<char>(o_y), pitch, width, B, cudaMemcpyDeviceToHost, hs.st));
  if ((r = hs.finish())) return r;
  for (int b = 0; b < B; ++b) memcpy(y + (size_t)b * y_pitch, hp + (size_t)b * pitch, nbytes[b]);
  return VTTS_OK;
}

// ---- per-slot stream ----------------------------------------------------------------------------------------------
// A slot carries its P mod block samples that no frame holds yet (as float, PCM-16 quantized when they are encoded), in
// one of two buffers that alternate push by push.  A push emits, per slot, the stream header with BEGIN, the frames its
// carried and new samples complete, and with END the short last frame.
struct vtts_flac_stream : StreamBase {
  int block, rate;
  RateCode rc;
  int nf;                          // frame slots per slot and push
  long long out_cap;               // bytes of a push's output buffer
  float* carry[2] = {nullptr, nullptr};
  int cur = 0;
  FrameDesc* desc = nullptr;
  FlacRow* d_rows = nullptr;
  RowOut* ro = nullptr;
  int* d_keep = nullptr;
  std::vector<FlacRow> rows;
  std::vector<int> keep;           // per slot (from, count) of the samples it carries after the push
  std::vector<int> carried;        // per slot: samples carried now
  std::vector<long long> frames;   // per slot: frames emitted since BEGIN
  vtts_flac_stream(vtts_ctx* c, int s, int f, int blk, int r, RateCode code)
      : StreamBase(c, s, f), block(blk), rate(r), rc(code), nf((blk - 1 + f + blk - 1) / blk),
        out_cap((long long)s * (HDR + (long long)((blk - 1 + f + blk - 1) / blk) * (FRAME_HDR_MAX + 1 + 2 + 2LL * blk))),
        rows(s), keep(2 * s), carried(s, 0), frames(s, 0) {}
  void carve(Arena& a) {
    carry[0] = a.take<float>((size_t)S * block);
    carry[1] = a.take<float>((size_t)S * block);
    desc = a.take<FrameDesc>((size_t)S * nf);
    d_rows = a.take<FlacRow>(S);
    ro = a.take<RowOut>(S);
    d_keep = a.take<int>(2 * (size_t)S);
  }
};

int vtts_flac_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, int block, vtts_flac_stream** out,
                            int64_t* out_bytes) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int r = create_check(ctx, "flac_stream_create", out, out_bytes != nullptr, max_streams, max_chunk_samples);
  if (r) return r;
  RateCode rc;
  if (!block_ok(block)) return ctx->fail(VTTS_ERR_BAD_ARG, "flac_stream_create: block %d (256, 512, 1024, 2048 or 4096)", block);
  if (!rate_code(rate, &rc)) return ctx->fail(VTTS_ERR_BAD_ARG, "flac_stream_create: rate %d has no FLAC frame-header code", rate);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_flac_stream> fs(new vtts_flac_stream(ctx, max_streams, max_chunk_samples, block, rate, rc));
  if ((long long)fs->out_cap > INT_MAX)
    return ctx->fail(VTTS_ERR_BAD_ARG, "flac_stream_create: a push's output of %lld bytes exceeds 2^31 - 1", fs->out_cap);
  r = stream_alloc(ctx, "flac_stream_create", *fs, [&](Arena& a) { fs->carve(a); });
  if (r) return r;
  *out_bytes = fs->out_cap;
  *out = fs.release();
  return VTTS_OK;
}

int vtts_flac_stream_destroy(vtts_ctx* ctx, vtts_flac_stream* fs) { return stream_destroy(ctx, "flac_stream_destroy", fs); }

int vtts_flac_stream_push(vtts_ctx* ctx, vtts_flac_stream* fs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                          uint8_t* y_dev, int32_t* tbl_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int r = stream_args(ctx, "flac_stream_push", fs, x_dev && n_new && flags && y_dev && tbl_dev);
  if (r) return r;
  if (overlaps(x_dev, (size_t)fs->S * fs->F * 4, y_dev, fs->out_cap) || overlaps(y_dev, fs->out_cap, tbl_dev, (size_t)fs->S * 8) ||
      overlaps(x_dev, (size_t)fs->S * fs->F * 4, tbl_dev, (size_t)fs->S * 8))
    return ctx->fail(VTTS_ERR_BAD_ARG, "flac_stream_push: the buffers overlap");
  const int B = fs->block;
  r = fs->slots.check(ctx, "flac_stream_push", fs->F, n_new, flags, [&](int s) {
    const long long c = (flags[s] & 1) ? 0 : fs->carried[s], m = c + n_new[s];
    const long long fr = ((flags[s] & 1) ? 0 : fs->frames[s]) + (m + B - 1) / B;
    return fr > 0x7FFFFFFFLL ? ctx->fail(VTTS_ERR_BAD_ARG, "flac_stream_push: slot %d passes frame number 2^31 - 1", s) : VTTS_OK;
  });
  if (r) return r;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  std::vector<long long> E1(fs->S);
  for (int s = 0; s < fs->S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = act && (flags[s] & 1), end = act && (flags[s] & 2);
    const int c = begin || !fs->slots.open[s] ? 0 : fs->carried[s], nn = act ? n_new[s] : 0, m = c + nn;
    const long long f0 = begin ? 0 : fs->frames[s];
    const int nfr = end ? (m + B - 1) / B : m / B, left = end ? 0 : m - nfr * B;
    fs->rows[s] = FlacRow{fs->carry[fs->cur] + (size_t)s * B, x_dev + (size_t)s * fs->F, c, m, nfr, begin ? 1 : 0, 0, f0, 0};
    fs->keep[2 * s] = nfr * B;
    fs->keep[2 * s + 1] = left;
    E1[s] = f0 + nfr;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // pageable sources: the call returns once they are staged, so the next push may rewrite them
  VTTS_CUDA(cudaMemcpyAsync(fs->d_rows, fs->rows.data(), fs->rows.size() * sizeof(FlacRow), cudaMemcpyHostToDevice, st));
  VTTS_CUDA(cudaMemcpyAsync(fs->d_keep, fs->keep.data(), fs->keep.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const FlacArgs A{fs->d_rows, fs->S, B, fs->rc, fs->rate, fs->nf, fs->desc, fs->ro, y_dev, 0, nullptr, tbl_dev};
  if ((r = flac_launch(ctx, A, st))) return r;
  flac_carry<<<fs->S, 256, 0, st>>>(fs->d_rows, fs->d_keep, B, fs->carry[1 - fs->cur]);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  for (int s = 0; s < fs->S; ++s) {
    if (!SlotState::active(n_new, flags, s) && !fs->slots.open[s]) continue;
    fs->carried[s] = fs->keep[2 * s + 1];
    if (SlotState::active(n_new, flags, s)) fs->frames[s] = E1[s];
  }
  fs->cur = 1 - fs->cur;
  fs->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_flac_stream_push_host(vtts_ctx* ctx, vtts_flac_stream* fs, const float* x, const int32_t* n_new, const uint8_t* flags,
                               uint8_t* y, int32_t* tbl) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int r = stream_args(ctx, "flac_stream_push_host", fs, x && n_new && flags && y && tbl);
  if (r) return r;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)fs->S * fs->F * 4), o_y = hs.out(fs->out_cap), o_t = hs.out((size_t)fs->S * 8, tbl);
  r = hs.run([&](cudaStream_t st) {
    return vtts_flac_stream_push(ctx, fs, hs.dev<const float>(o_x), n_new, flags, hs.dev<uint8_t>(o_y), hs.dev<int32_t>(o_t), st);
  });
  if (r) return r;
  long long total = 0;   // the slots' bytes lie one after another from the start of the buffer
  for (int s = 0; s < fs->S; ++s) total += tbl[2 * s + 1];
  if (total) r = hs.fetch(o_y, y, (size_t)total);
  return r ? r : hs.finish();
}
