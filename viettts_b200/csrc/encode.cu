// Wire encodings of synthesized audio: PCM-16 and G.711 mu-law / A-law, and their expansion back to float32
// (oracle/g711_oracle.py is the integer definition; the device output equals it bit for bit in every vtts_precision mode).
//
// Encode, per sample x: v = clip(rint(x * 32767), -32768, 32767) with the product in double (exact for every float) and
// round-half-to-even; NaN gives 0, +-Inf clip.  pcm16 stores v; mu-law codes the 14-bit v >> 2 and A-law the 13-bit
// v >> 3 by the G.711 segment rules, the segment found from the bit length of the biased magnitude (no tables).
// Decode: the G.711 expansion to int16, then v / 32767 as an IEEE fp32 division.
//
// Both kernels are elementwise: one launch, grid (groups / 256, B), one thread per group of V = 4 samples of a row.  A
// row's group 0 holds its first h < 4 samples, so that the groups after it start where both the row's input and output
// are 4-element aligned and move as one 16-byte float4 and one 4- or 8-byte code vector.  A row whose input and output
// addresses reach that alignment at different samples (a caller's offset view) runs every group element by element.
#include <type_traits>

#include "pcm16.cuh"
#include "stream_common.cuh"

namespace {

constexpr int V = 4;
constexpr int THREADS = 256;

template <int E>
using Code = std::conditional_t<E == VTTS_ENC_PCM16, int16_t, uint8_t>;
template <int E>
using CodeVec = std::conditional_t<E == VTTS_ENC_PCM16, short4, uchar4>;

template <int E>
__device__ __forceinline__ Code<E> silence() {
  return (Code<E>)(E == VTTS_ENC_PCM16 ? 0 : (E == VTTS_ENC_ULAW ? 0xFF : 0xD5));
}

__device__ __forceinline__ int bit_length(int p) { return 32 - __clz(p); }

template <int E>
__device__ __forceinline__ Code<E> encode_one(float x) {
  const int v = VTTS_PCM16_OF(x);
  if (E == VTTS_ENC_PCM16) return (Code<E>)v;
  if (E == VTTS_ENC_ULAW) {
    int p = v >> 2, mask = 0xFF;
    if (p < 0) p = -p, mask = 0x7F;
    p = min(p, 8159) + 33;
    const int seg = max(bit_length(p) - 6, 0);   // the first seg with p <= 2^(6 + seg) - 1
    return (Code<E>)((seg >= 8 ? 0x7F : (seg << 4 | ((p >> (seg + 1)) & 0xF))) ^ mask);
  }
  int p = v >> 3, mask = 0xD5;
  if (p < 0) p = -p - 1, mask = 0x55;
  const int seg = max(bit_length(p) - 5, 0);     // the first seg with p <= 2^(5 + seg) - 1
  return (Code<E>)((seg >= 8 ? 0x7F : (seg << 4 | ((seg < 2 ? p >> 1 : p >> seg) & 0xF))) ^ mask);
}

template <int E>
__device__ __forceinline__ float decode_one(Code<E> c) {
  int v;
  if (E == VTTS_ENC_PCM16) {
    v = c;
  } else if (E == VTTS_ENC_ULAW) {
    const int u = ~(int)c & 0xFF, t = (((u & 0xF) << 3) + 0x84) << ((u & 0x70) >> 4);
    v = u & 0x80 ? 0x84 - t : t - 0x84;
  } else {
    const int a = (int)c ^ 0x55, seg = (a & 0x70) >> 4;
    const int t = (((a & 0xF) << 4) + (seg ? 0x108 : 8)) << max(seg - 1, 0);
    v = a & 0x80 ? t : -t;
  }
  return (float)v / 32767.0f;
}

// the first sample h < V from which both rows are V-element aligned, or -1 when they never are at the same sample
template <class A, class B>
__device__ __forceinline__ int aligned_head(const A* a, const B* b) {
  const uintptr_t ua = (uintptr_t)a, ub = (uintptr_t)b;
  if (ua % sizeof(A) || ub % sizeof(B)) return -1;
  const int pa = (int)(ua / sizeof(A) % V), pb = (int)(ub / sizeof(B) % V);
  return pa == pb ? (V - pa) % V : -1;
}

// samples [lo, hi) of group g of a row of S samples, and whether it moves as one vector
struct Group {
  long long lo, hi;
  bool vec;
};
__device__ __forceinline__ Group row_group(int h, int S) {
  const long long g = (long long)blockIdx.x * THREADS + threadIdx.x;
  const int h0 = max(h, 0);
  const long long lo = g == 0 ? 0 : h0 + V * (g - 1), hi = min(g == 0 ? (long long)h0 : h0 + V * g, (long long)S);
  return {lo, hi, h >= 0 && g > 0 && hi - lo == V};
}

template <int E>
__global__ void __launch_bounds__(THREADS) encode_kernel(const float* __restrict__ x, const int* __restrict__ n_in, int S,
                                                         Code<E>* __restrict__ y) {
  const int b = blockIdx.y;
  const float* xr = x + (long long)b * S;
  Code<E>* yr = y + (long long)b * S;
  const int n = n_in ? min(max(n_in[b], 0), S) : S;
  const Group gr = row_group(aligned_head(xr, yr), S);
  if (gr.vec) {
    const float4 v = *reinterpret_cast<const float4*>(xr + gr.lo);
    const long long t = gr.lo;
    CodeVec<E> c;
    c.x = t < n ? encode_one<E>(v.x) : silence<E>();
    c.y = t + 1 < n ? encode_one<E>(v.y) : silence<E>();
    c.z = t + 2 < n ? encode_one<E>(v.z) : silence<E>();
    c.w = t + 3 < n ? encode_one<E>(v.w) : silence<E>();
    *reinterpret_cast<CodeVec<E>*>(yr + gr.lo) = c;
    return;
  }
  for (long long t = gr.lo; t < gr.hi; ++t) yr[t] = t < n ? encode_one<E>(xr[t]) : silence<E>();
}

template <int E>
__global__ void __launch_bounds__(THREADS) decode_kernel(const Code<E>* __restrict__ c, const int* __restrict__ n_in, int S,
                                                         float* __restrict__ y) {
  const int b = blockIdx.y;
  const Code<E>* cr = c + (long long)b * S;
  float* yr = y + (long long)b * S;
  const int n = n_in ? min(max(n_in[b], 0), S) : S;
  const Group gr = row_group(aligned_head(cr, yr), S);
  if (gr.vec) {
    const CodeVec<E> v = *reinterpret_cast<const CodeVec<E>*>(cr + gr.lo);
    const long long t = gr.lo;
    float4 o;
    o.x = t < n ? decode_one<E>(v.x) : 0.f;
    o.y = t + 1 < n ? decode_one<E>(v.y) : 0.f;
    o.z = t + 2 < n ? decode_one<E>(v.z) : 0.f;
    o.w = t + 3 < n ? decode_one<E>(v.w) : 0.f;
    *reinterpret_cast<float4*>(yr + gr.lo) = o;
    return;
  }
  for (long long t = gr.lo; t < gr.hi; ++t) yr[t] = t < n ? decode_one<E>(cr[t]) : 0.f;
}

size_t code_bytes(int encoding) { return encoding == VTTS_ENC_PCM16 ? 2 : 1; }

// the encoding and batch shape of a call of entry point `who`
int coder_args(vtts_ctx* ctx, const char* who, int B, int S, int encoding) {
  if (encoding != VTTS_ENC_PCM16 && encoding != VTTS_ENC_ULAW && encoding != VTTS_ENC_ALAW)
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: encoding %d (VTTS_ENC_PCM16, _ULAW or _ALAW)", who, encoding);
  return batch_check(ctx, who, B, S, S_ANY);
}

// both buffers given and apart
int coder_apart(vtts_ctx* ctx, const char* who, const void* f32, const void* codes, int B, int S, int encoding) {
  if (!f32 || !codes) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
  const uintptr_t a = (uintptr_t)f32, c = (uintptr_t)codes;
  const size_t n = (size_t)B * S;
  if (a < c + n * code_bytes(encoding) && c < a + n * 4) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: the output overlaps the input", who);
  return VTTS_OK;
}

dim3 coder_grid(int B, int S) {
  const long long groups = 1 + (S + V - 1) / V;   // group 0 (the aligned head) and at most ceil(S / V) after it
  return dim3((unsigned)((groups + THREADS - 1) / THREADS), (unsigned)B);
}

int encode_launch(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int encoding, void* y, cudaStream_t st) {
  const dim3 grid = coder_grid(B, S);
  if (encoding == VTTS_ENC_PCM16)
    encode_kernel<VTTS_ENC_PCM16><<<grid, THREADS, 0, st>>>(x, n_in, S, (int16_t*)y);
  else if (encoding == VTTS_ENC_ULAW)
    encode_kernel<VTTS_ENC_ULAW><<<grid, THREADS, 0, st>>>(x, n_in, S, (uint8_t*)y);
  else
    encode_kernel<VTTS_ENC_ALAW><<<grid, THREADS, 0, st>>>(x, n_in, S, (uint8_t*)y);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

int decode_launch(vtts_ctx* ctx, const void* c, const int32_t* n_in, int B, int S, int encoding, float* y, cudaStream_t st) {
  const dim3 grid = coder_grid(B, S);
  if (encoding == VTTS_ENC_PCM16)
    decode_kernel<VTTS_ENC_PCM16><<<grid, THREADS, 0, st>>>((const int16_t*)c, n_in, S, y);
  else if (encoding == VTTS_ENC_ULAW)
    decode_kernel<VTTS_ENC_ULAW><<<grid, THREADS, 0, st>>>((const uint8_t*)c, n_in, S, y);
  else
    decode_kernel<VTTS_ENC_ALAW><<<grid, THREADS, 0, st>>>((const uint8_t*)c, n_in, S, y);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace

int vtts_encode(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int encoding, void* y_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = coder_args(ctx, "encode", B, S, encoding);
  if (!rc) rc = coder_apart(ctx, "encode", x_dev, y_dev, B, S, encoding);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return encode_launch(ctx, x_dev, n_dev, B, S, encoding, y_dev, (cudaStream_t)stream);
}

int vtts_encode_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int encoding, void* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = coder_args(ctx, "encode_host", B, S, encoding);
  if (!rc) rc = coder_apart(ctx, "encode_host", x, y, B, S, encoding);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("encode_host", x, n_in, B, S);
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * S * code_bytes(encoding), y);
  return hs.run([&](cudaStream_t st) { return encode_launch(ctx, hs.x(), hs.n(), B, S, encoding, hs.dev<void>(o_y), st); });
}

int vtts_decode(vtts_ctx* ctx, const void* c_dev, const int32_t* n_dev, int B, int S, int encoding, float* y_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = coder_args(ctx, "decode", B, S, encoding);
  if (!rc) rc = coder_apart(ctx, "decode", y_dev, c_dev, B, S, encoding);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return decode_launch(ctx, c_dev, n_dev, B, S, encoding, y_dev, (cudaStream_t)stream);
}

int vtts_decode_host(vtts_ctx* ctx, const void* c, const int32_t* n_in, int B, int S, int encoding, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = coder_args(ctx, "decode_host", B, S, encoding);
  if (!rc) rc = coder_apart(ctx, "decode_host", y, c, B, S, encoding);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("decode_host", c, n_in, B, S, true, code_bytes(encoding));
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return decode_launch(ctx, hs.x<void>(), hs.n(), B, S, encoding, hs.dev<float>(o_y), st); });
}
