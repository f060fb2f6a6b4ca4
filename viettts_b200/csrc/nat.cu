// NAT acoustic model forward -- restates AcousticModel.inference
// (vietTTS/nat/model.py:123-144) with batch semantics "row b == reference run on row b alone".
//
//   TokenEncoder            model.py:26-47   embed_kernel, generic conv (+BN+relu), lstm_scan_kernel
//   upsample                model.py:102-111 upsample_kernel
//   loop_fn (AR decoder)    model.py:129-142 decoder_scan_kernel  (persistent, cooperative)
//   postnet + residual      model.py:113-121,143-144 generic conv (+BN+tanh)
//
// Recurrent kernels: one cooperative grid of 128 CTAs; CTA c owns 4 hidden units of every LSTM
// layer (16 gate columns i,g,f,o) and keeps that slice of the RECURRENT weights resident in
// shared memory for the whole scan; the input projections that do not depend on the recurrence
// (token embedding path for the encoder, cond_t for the decoder) are hoisted into one GEMM
// before the scan (generic conv kernel with k=1).  State vectors live in global memory (L2) and
// are exchanged with one grid barrier per dependent phase.
#include <cooperative_groups.h>

#include "threefry.cuh"
#include "vtts_internal.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int SCAN_CTAS = 128;
constexpr int SCAN_THREADS = 256;
constexpr int UPC = 4;        // hidden units per CTA per layer
constexpr int NCOL = 16;      // 4 gates x UPC
constexpr int RG = 8;         // batch rows per register tile
constexpr int NSLICE = 64;    // K slices (SCAN_THREADS / 4 column groups)
constexpr int MAX_ROWS = 128; // batch rows per scan launch

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// jax split(key) in the classic layout: (next key, sub-key) = ((a0, b0), (a1, b1)) with (a0, a1) = threefry(key, (0, 2)),
// (b0, b1) = threefry(key, (1, 3)); one hk.next_rng_key() call returns the sub-key
__host__ __device__ inline void jax_split(uint32_t& k0, uint32_t& k1, uint32_t& s0, uint32_t& s1) {
  uint32_t a0, a1, b0, b1;
  threefry2x32(k0, k1, 0u, 2u, a0, a1);
  threefry2x32(k0, k1, 1u, 3u, b0, b1);
  k0 = a0; k1 = b0; s0 = a1; s1 = b1;
}

// The one threefry evaluation per mask element of the two on-device streams.
//   SEED       key (lo, hi) = seed, counter (frame, row << 12 | entry), output 0: a row's stream depends on its row index
//              in the call and the absolute frame, not on the padded frame count of the batch it happens to share.
//   REFERENCE  word i of jax random_bits(rkey, n) in the classic layout (n even): i < n/2 is output 0 of
//              threefry(rkey, (i, i + n/2)), i >= n/2 is output 1 of threefry(rkey, (i - n/2, i)).
__device__ __forceinline__ uint32_t stream_word(int mode, uint64_t seed, int b, int t, uint32_t entry, uint2 rkey, uint32_t ri, uint32_t rn) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32), c0 = (uint32_t)t, c1 = ((uint32_t)b << 12) | entry;
  bool hi = false;
  if (mode == VTTS_DROPOUT_REFERENCE) {
    const uint32_t h = rn >> 1;
    hi = ri >= h;
    k0 = rkey.x; k1 = rkey.y; c0 = hi ? ri - h : ri; c1 = c0 + h;
  }
  uint32_t o0, o1;
  threefry2x32(k0, k1, c0, c1, o0, o1);
  return hi ? o1 : o0;
}

// prenet dropout scale of (row b, frame t, layer, unit); rkey / ri / rn: the REFERENCE draw this element belongs to
__device__ __forceinline__ float keep_scale(int mode, const uint8_t* keep, uint64_t seed, int b, int t, int N, int layer, int unit,
                                            uint2 rkey = make_uint2(0u, 0u), uint32_t ri = 0u, uint32_t rn = 0u) {
  if (mode == VTTS_DROPOUT_OFF) return 1.f;
  if (mode == VTTS_DROPOUT_MASK) return keep[(((size_t)b * N + t) * 2 + layer) * vc::PRENET + unit] ? 2.f : 0.f;
  // bernoulli(0.5) keeps where the word is below 2^31, in both streams
  return stream_word(mode, seed, b, t, (uint32_t)(layer * vc::PRENET + unit), rkey, ri, rn) < 0x80000000u ? 2.f : 0.f;
}

// Autoregressive scan, REFERENCE: every row draws what the reference draws for a batch of one -- frame t, layer l uses
// sub-key 2t + l of the chain (ref_subkey_chain_kernel) and bernoulli(sub, 0.5, [1,256])
__device__ __forceinline__ float ar_keep_scale(int mode, const uint8_t* keep, uint64_t seed, const uint2* subkeys, int b, int t, int N,
                                               int layer, int unit) {
  const uint2 rk = mode == VTTS_DROPOUT_REFERENCE ? subkeys[2 * t + layer] : make_uint2(0u, 0u);
  return keep_scale(mode, keep, seed, b, t, N, layer, unit, rk, (uint32_t)unit, (uint32_t)vc::PRENET);
}

// Teacher-forced pass, REFERENCE: the reference draws over the whole batch, bernoulli(key_l, 0.5, [B,N,256]) per layer;
// b is the row in the call and B its row count (B * N * 512 < 2^32 is checked by the host)
__device__ __forceinline__ float tf_keep_scale(int mode, const uint8_t* keep, uint64_t seed, uint2 rkey, int b, int t, int B, int N,
                                               int layer, int unit) {
  return keep_scale(mode, keep, seed, b, t, N, layer, unit, rkey, ((uint32_t)b * N + t) * vc::PRENET + unit, (uint32_t)B * N * vc::PRENET);
}

// Sub-keys 0 .. n-1 of the hk.next_rng_key() chain from key (seed >> 32, (uint32)seed), as uint32 pairs.  The chain is
// sequential: one thread walks it (two independent threefry evaluations per step).
__global__ void ref_subkey_chain_kernel(uint64_t seed, int n, uint2* __restrict__ out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  uint32_t k0 = (uint32_t)(seed >> 32), k1 = (uint32_t)seed;
  for (int i = 0; i < n; ++i) {
    uint32_t s0, s1;
    jax_split(k0, k1, s0, s1);
    out[i] = make_uint2(s0, s1);
  }
}

// ---- small kernels ---------------------------------------------------------------------------------
__global__ void embed_kernel(const int32_t* __restrict__ tokens, const float* __restrict__ emb, float* __restrict__ out, int n_tok) {
  // out[tok][256] = emb[tokens[tok]][256]
  const int tok = blockIdx.x * 4 + threadIdx.x / 64;
  if (tok >= n_tok) return;
  int id = tokens[tok];
  id = id < 0 ? 0 : (id >= vc::VOCAB ? vc::VOCAB - 1 : id);
  const int c4 = (threadIdx.x % 64) * 4;
  *reinterpret_cast<float4*>(out + (size_t)tok * vc::ENC_D + c4) = __ldg(reinterpret_cast<const float4*>(emb + (size_t)id * vc::ENC_D + c4));
}

// dst[c][r][q] = src[(row0 + r)*ld + (q / upc)*gate_stride + c*upc + (q % upc)]
__global__ void repack_cols_kernel(const float* __restrict__ src, int ld, int row0, int nrows, float* __restrict__ dst,
                                   int ncta, int ncols, int upc, int gate_stride) {
  const size_t total = (size_t)ncta * nrows * ncols;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int q = idx % ncols;
    int r = (idx / ncols) % nrows;
    int c = idx / ((size_t)ncols * nrows);
    int col = (q / upc) * gate_stride + c * upc + (q % upc);
    dst[idx] = src[(size_t)(row0 + r) * ld + col];
  }
}

// ---- Gaussian upsampling (model.py:102-111) --------------------------------------------------------
// out[b,n,:] = sum_l softmax_l(-(mid_l - n)^2/10) enc[b,l,:],  mid = cumsum(dur) - dur/2
constexpr int UP_F = 8;  // frames per CTA
__global__ void __launch_bounds__(256) upsample_kernel(const float* __restrict__ enc, const float* __restrict__ dur,
                                                       const int32_t* __restrict__ lengths, const int32_t* __restrict__ n_frames,
                                                       int L, int N, float* __restrict__ out, int out_ld) {
  extern __shared__ float sm[];
  float* mid = sm;            // [L]
  float* w = sm + L;          // [UP_F][L]
  const int b = blockIdx.y, f0 = blockIdx.x * UP_F, tid = threadIdx.x;
  const int len = lengths ? min(lengths[b], L) : L;
  const int nf = n_frames ? min(n_frames[b], N) : N;
  if (f0 >= nf) return;
  if (tid < 32) {
    // sequential cumsum in fp32 (jnp.cumsum), done by one warp with a carried scan
    float carry = 0.f;
    for (int l0 = 0; l0 < len; l0 += 32) {
      int l = l0 + tid;
      float d = l < len ? dur[(size_t)b * L + l] : 0.f;
      float s = d;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        float v = __shfl_up_sync(0xffffffffu, s, o);
        if (tid >= o) s += v;
      }
      s += carry;
      if (l < len) mid[l] = s - d / 2.f;
      carry = __shfl_sync(0xffffffffu, s, 31);
    }
  }
  __syncthreads();
  const int warp = tid / 32, lane = tid % 32;  // 8 warps = UP_F frames
  {
    const float n = (float)(f0 + warp);
    float mx = -INFINITY;
    for (int l = lane; l < len; l += 32) {
      float d = mid[l] - n;
      float v = -(d * d) / 10.0f;
      w[warp * L + l] = v;
      mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float s = 0.f;
    for (int l = lane; l < len; l += 32) {
      float e = expf(w[warp * L + l] - mx);
      w[warp * L + l] = e;
      s += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int l = lane; l < len; l += 32) w[warp * L + l] = w[warp * L + l] / s;  // jax.nn.softmax: exp / sum
  }
  __syncthreads();
  // each thread: 2 channels x UP_F frames
  float acc[UP_F][2];
#pragma unroll
  for (int f = 0; f < UP_F; ++f) acc[f][0] = acc[f][1] = 0.f;
  const float* e = enc + (size_t)b * L * vc::ENC_OUT + tid * 2;
  for (int l = 0; l < len; ++l) {
    const float2 x = __ldg(reinterpret_cast<const float2*>(e + (size_t)l * vc::ENC_OUT));
#pragma unroll
    for (int f = 0; f < UP_F; ++f) {
      const float ww = w[f * L + l];
      acc[f][0] = fmaf(ww, x.x, acc[f][0]);
      acc[f][1] = fmaf(ww, x.y, acc[f][1]);
    }
  }
#pragma unroll
  for (int f = 0; f < UP_F; ++f) {
    const int n = f0 + f;
    if (n < nf) {
      float2 o = make_float2(acc[f][0], acc[f][1]);
      *reinterpret_cast<float2*>(out + ((size_t)b * N + n) * out_ld + tid * 2) = o;
    }
  }
}

// ---- shared device pieces of the scan kernels -------------------------------------------------------
struct Seg {
  const float* p;   // p[row*stride + i]
  int n;            // multiple of 4
  int stride;
};

// LSTM cell update for (row r, unit uu) from zs (hk.LSTM: i,g,f,o; forget bias +1)
__device__ __forceinline__ float lstm_cell(const float* zs, int r, int uu, float zadd_i, float zadd_g, float zadd_f, float zadd_o, float& c) {
  const float zi = zs[r * NCOL + 0 * UPC + uu] + zadd_i;
  const float zg = zs[r * NCOL + 1 * UPC + uu] + zadd_g;
  const float zf = zs[r * NCOL + 2 * UPC + uu] + zadd_f;
  const float zo = zs[r * NCOL + 3 * UPC + uu] + zadd_o;
  const float f = sigmoidf_(zf + 1.f);
  c = f * c + sigmoidf_(zi) * tanhf(zg);
  return sigmoidf_(zo) * tanhf(c);
}

// ---- encoder BiLSTM scan (model.py:36-46) ---------------------------------------------------------
struct EncScanArgs {
  const float* zx;        // [2][B][L][1024] hoisted x.Wx + b per direction
  const float* whr;       // [2][64][256][16] recurrent weights, per direction / CTA
  const int32_t* lengths; // [B] or null
  float* out;             // [B][L][512]  (fwd | bwd)
  int B, L;
};

// ---- autoregressive decoder scan (model.py:129-142) ------------------------------------------------
// One cooperative grid of 128 CTAs, up to 128 batch rows per launch (row groups of 32).  CTA c owns
//   * 4 hidden units (16 gate columns) of both LSTM layers; its slices of the recurrent matrices (768x16 + 1280x16
//     fp32) live in REGISTERS;
//   * prenet columns 2c and 2c+1 of p1 = drop(relu([h0,h1]_{t-1}.(Wo.W1) + bo.W1)) and of p2 = drop(relu(p1.W2));
//     those weight slices (1024x2 + 256x2 fp32) live in SHARED memory.
// A persistent shared-memory buffer holds [p2 | h0 | h1] of one row group.  A frame has four dependent exchanges
// through L2, each closed by a grid barrier split into arrive and wait (dec_arrive / dec_wait):
//   A  p1(t) from [h0 | h1]_{t-1}        arrive; zp1 = h1_{t-1}.W1[h1 rows], prefetch zc0[t] / zc1[t]; wait
//   B  p2(t) from p1(t)                  arrive; wait
//   C  LSTM0: h0_t                       arrive; wait
//   D  LSTM1: h1_t                       arrive; zp0 = h0_t.W0[h0 rows] for frame t+1; wait
// so the products of the state that is already final run while the barrier is open instead of on the critical path
// (with more than one row group, the last group's only; the others are computed inline while their rows are staged).
// The output projection mel_t = [h0,h1]_t.Wo + bo is NOT part of the scan: nothing in the recurrence reads mel_t
// (the prenet consumes the precomposed Wo.W1), so every frame's [h0 | h1] is written to `hout` and one GEMM
// projects the whole sequence afterwards.
struct DecScanArgs {
  const float* zc0;      // [B][N][2048] cond.W0[0:512] + b0
  const float* zc1;      // [B][N][2048] cond.W1[0:512] + b1
  const float* w0r;      // [128][768][16]   rows 512..1279 of lstm0   ([p2, h0])
  const float* w1r;      // [128][1280][16]  rows 512..1791 of lstm1   ([p2, h0, h1])
  const float* wc;       // [128][1024][2]   (Wo . W1) columns 2c, 2c+1 per CTA
  const float* bc;       // [256]            bo . W1
  const float* wp2;      // [128][256][2]    prenet fc2 columns 2c, 2c+1 per CTA
  const uint8_t* keep;   // [B][N][2][256] or null (indexed with row_base)
  const uint2* subkeys;  // [N][2] REFERENCE sub-keys of the frames' two prenet draws, or null
  uint64_t seed;
  int mode;
  float* p1;             // [B][256]
  float* p2;             // [B][256]
  float* h0;             // [2][B][512] compact double-buffered state the recurrence reads (frame parity)
  float* h1;             // [2][B][512]
  unsigned int* bar;     // arrival counter of the split grid barriers (zeroed before the launch)
  int* err;              // device int set before trapping on a barrier time-out
  float* hout;           // [B][N][1024] decoder outputs [h0_t | h1_t] of every frame (write only): the output projection
                         // runs over the whole tensor as ONE GEMM after the scan
  int B, N;              // rows of this launch (<= 128), frames
  int row_base;          // first row of this launch inside the full batch (dropout stream indexing)
  int N_total_rows;      // unused
  long long* dbg;        // optional per-CTA phase timers [grid][16]
  // RESUME instantiation only (acoustic_stream.cu): launch row r advances stream slot rows[r].x from absolute frame
  // rows[r].y by rows[r].z <= N steps (N = the largest); zc0 / zc1 / keep are per slot [S][zstride][...], the dropout
  // row is the slot, and hout is [B][hstride][1024] by local step
  const int4* rows;      // [B] (slot, t0, n, -)
  float* state;          // [S][4][512] carried h0, c0, h1, c1 of every slot: loaded at launch start, stored after a row's last step
  int zstride;           // frames per slot of zc0 / zc1 / keep (the stream's max_frames)
  int hstride;           // frames per row of hout (the stream's max_chunk_frames)
};

constexpr int DEC_XR = 32;                 // batch rows per staging group (smem holds the state of one group)
constexpr int DEC_NG = 4;                  // row groups per launch: up to 128 rows share the four barriers of a frame
constexpr int DEC_KPAD = vc::PRENET + 2 * vc::DEC_H + 4;   // 1284: [p2 | h0 | h1] + pad
// a cooperative grid must be co-resident: one CTA per SM, 128 of the 132 SMs of an H100 SXM
constexpr int DEC_CTAS = 128;
constexpr int DEC_PCOL = vc::PRENET / DEC_CTAS;   // 2 prenet columns per CTA

// copy rows [0,nr) x [n floats] of a global matrix (row stride `stride`) into smem (row pitch `pitch`, column
// offset koff); p == nullptr writes zeros.  8 x 16 B loads in flight per thread.
__device__ __forceinline__ void dec_fetch(float* xs, int pitch, int koff, const float* p, int n, int stride, int nr) {
  const int n4 = n >> 2;
  const int total = nr * n4;
  for (int e0 = threadIdx.x; e0 < total; e0 += SCAN_THREADS * 8) {
    float4 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int e = e0 + u * SCAN_THREADS;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (e < total && p) {
        const int r = e / n4, i4 = (e - r * n4) * 4;
        v[u] = __ldcg(reinterpret_cast<const float4*>(p + (size_t)r * stride + i4));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int e = e0 + u * SCAN_THREADS;
      if (e < total) {
        const int r = e / n4, i4 = (e - r * n4) * 4;
        *reinterpret_cast<float4*>(xs + (size_t)r * pitch + koff + i4) = v[u];
      }
    }
  }
}

// same copy with cp.async (16 B, L2 only): the data goes global -> shared without passing through registers, so a fetch
// can stay in flight while the CTA computes on operands that have already arrived (decoder_tf_scan_kernel)
__device__ __forceinline__ void dec_fetch_async(float* xs, int pitch, int koff, const float* p, int n, int stride, int nr) {
  const int n4 = n >> 2;
  const int total = nr * n4;
  for (int e = threadIdx.x; e < total; e += SCAN_THREADS) {
    const int r = e / n4, i4 = (e - r * n4) * 4;
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(xs + (size_t)r * pitch + koff + i4);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(p + (size_t)r * stride + i4) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// acc[8 rows][4 cols] partial sums over this thread's K slice -> butterfly over the 8 slices of the
// warp (28 shuffles); afterwards the thread holds the warp-level sums of row (lane>>2), cols cg*4..+3.
__device__ __forceinline__ float4 warp_reduce_rows(float (&acc)[RG][4], int lane) {
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
  float a4[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float send = b4 ? acc[r][c] : acc[r + 4][c];
      const float keep = b4 ? acc[r + 4][c] : acc[r][c];
      a4[r][c] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  float a2[2][4];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float send = b3 ? a4[r][c] : a4[r + 2][c];
      const float keep = b3 ? a4[r + 2][c] : a4[r][c];
      a2[r][c] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
  float a1[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float send = b2 ? a2[0][c] : a2[1][c];
    const float keep = b2 ? a2[1][c] : a2[0][c];
    a1[c] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  return make_float4(a1[0], a1[1], a1[2], a1[3]);
}

// partial LSTM pre-activations for the staged rows: zout[row][16] = xs[row][0:64*SL] . w  (+ zadd[row][16])
// (xs already points at the first column of the K segment; thread (ks, cg) owns rows ks*SL.. of the segment)
template <int SL, int PITCH = DEC_KPAD>
__device__ __forceinline__ void dec_matmul(const float* __restrict__ xs, const float (&w)[SL][4], int ngroups, float* part, float* zout,
                                           const float* zadd) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ks = tid >> 2;
  for (int g = 0; g < ngroups; ++g) {
    float acc[RG][4];
#pragma unroll
    for (int r = 0; r < RG; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
    const float* xk = xs + (size_t)(g * RG) * PITCH + ks * SL;
#pragma unroll
    for (int kk = 0; kk < SL; kk += 4) {
#pragma unroll
      for (int r = 0; r < RG; ++r) {
        const float4 xv = *reinterpret_cast<const float4*>(xk + (size_t)r * PITCH + kk);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          acc[r][c] = fmaf(xv.x, w[kk + 0][c], acc[r][c]);
          acc[r][c] = fmaf(xv.y, w[kk + 1][c], acc[r][c]);
          acc[r][c] = fmaf(xv.z, w[kk + 2][c], acc[r][c]);
          acc[r][c] = fmaf(xv.w, w[kk + 3][c], acc[r][c]);
        }
      }
    }
    const float4 s = warp_reduce_rows(acc, lane);
    *reinterpret_cast<float4*>(part + ((size_t)warp * DEC_XR + g * RG + (lane >> 2)) * NCOL + (lane & 3) * 4) = s;
  }
  __syncthreads();
  for (int o = tid; o < ngroups * RG * NCOL; o += SCAN_THREADS) {
    float s = zadd ? zadd[o] : 0.f;
#pragma unroll
    for (int wv = 0; wv < SCAN_THREADS / 32; ++wv) s += part[(size_t)wv * DEC_XR * NCOL + o];
    zout[o] = s;
  }
  __syncthreads();
}

// ---- encoder BiLSTM scan (model.py:36-46) ---------------------------------------------------------
__global__ void __launch_bounds__(SCAN_THREADS, 1) enc_scan_kernel(const EncScanArgs a) {
  // 128 CTAs: direction = cta / 64; CTA owns 4 hidden units (16 gate columns); its 256x16 slice of the recurrent
  // matrix lives in registers (4 rows x 4 columns per thread); h_{t-1} of up to 32 rows is staged per step.
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) float sm[];
  constexpr int K = vc::ENC_D, H = vc::ENC_D, XP = K + 4, SL = K / NSLICE;   // 256, 256, 260, 4
  float* xs = sm;                                // [32][XP]
  float* part = xs + 32 * XP;                    // [8][32][16]
  float* zs = part + 8 * DEC_XR * NCOL;          // [32][16]
  float* cst = zs + DEC_XR * NCOL;               // [MAX_ROWS][UPC]
  __shared__ int zero_row[DEC_XR];
  const int dir = blockIdx.x / 64, c = blockIdx.x % 64, tid = threadIdx.x;
  const int ks = tid >> 2, cgp = tid & 3;
  const int B = a.B, L = a.L;
  float wh[SL][4];
  {
    const float* g = a.whr + (((size_t)dir * 64 + c) * K + ks * SL) * NCOL + cgp * 4;
#pragma unroll
    for (int i = 0; i < SL; ++i) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(g + (size_t)i * NCOL));
      wh[i][0] = v.x; wh[i][1] = v.y; wh[i][2] = v.z; wh[i][3] = v.w;
    }
  }
  for (int e = tid; e < MAX_ROWS * UPC; e += SCAN_THREADS) cst[e] = 0.f;
  for (int e = tid; e < 32 * XP; e += SCAN_THREADS) xs[e] = 0.f;
  __syncthreads();
  for (int s = 0; s < L; ++s) {
    const int t = dir == 0 ? s : L - 1 - s;
    const int tprev = dir == 0 ? t - 1 : t + 1;
    for (int row0 = 0; row0 < B; row0 += DEC_XR) {
      const int nr = min(DEC_XR, B - row0);
      if (tid < DEC_XR) {
        int z = 1;
        if (tid < nr) {
          const int len = a.lengths ? min(a.lengths[row0 + tid], L) : L;
          // fwd: zero state at t=0.  bwd: ResetCore mask = (t >= len-1) (model.py:37,40)
          z = dir == 0 ? (s == 0) : (s == 0 || t >= len - 1);
        }
        zero_row[tid] = z;
      }
      __syncthreads();
      // stage h_{t-1} (zero for reset rows)
      for (int e = tid; e < nr * (H / 4); e += SCAN_THREADS) {
        const int r = e / (H / 4), i4 = (e - r * (H / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!zero_row[r]) v = __ldcg(reinterpret_cast<const float4*>(a.out + ((size_t)(row0 + r) * L + tprev) * vc::ENC_OUT + dir * H + i4));
        *reinterpret_cast<float4*>(xs + (size_t)r * XP + i4) = v;
      }
      __syncthreads();
      dec_matmul<SL, XP>(xs, wh, (nr + RG - 1) / RG, part, zs, nullptr);
      if (tid < nr * UPC) {
        const int r = tid / UPC, uu = tid % UPC, b = row0 + r;
        const float* zx = a.zx + (((size_t)dir * B + b) * L + t) * (4 * H) + c * UPC + uu;
        float cc = zero_row[r] ? 0.f : cst[b * UPC + uu];
        const float h = lstm_cell(zs, r, uu, __ldg(zx), __ldg(zx + H), __ldg(zx + 2 * H), __ldg(zx + 3 * H), cc);
        cst[b * UPC + uu] = cc;
        a.out[((size_t)b * L + t) * vc::ENC_OUT + dir * H + c * UPC + uu] = h;
      }
      __syncthreads();
    }
    grid.sync();
  }
}

// same, accumulating two K segments (xa: 64*SLA columns with weights wa; xb: 64*SLB columns with wb) before ONE reduction
template <int SLA, int SLB, int PITCH = DEC_KPAD>
__device__ __forceinline__ void dec_matmul2(const float* __restrict__ xa, const float (&wa)[SLA][4], const float* __restrict__ xb,
                                            const float (&wb)[SLB][4], int ngroups, float* part, float* zout, const float* zadd) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ks = tid >> 2;
  for (int g = 0; g < ngroups; ++g) {
    float acc[RG][4];
#pragma unroll
    for (int r = 0; r < RG; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
    const float* xk = xa + (size_t)(g * RG) * PITCH + ks * SLA;
#pragma unroll
    for (int kk = 0; kk < SLA; kk += 4) {
#pragma unroll
      for (int r = 0; r < RG; ++r) {
        const float4 xv = *reinterpret_cast<const float4*>(xk + (size_t)r * PITCH + kk);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          acc[r][c] = fmaf(xv.x, wa[kk + 0][c], acc[r][c]);
          acc[r][c] = fmaf(xv.y, wa[kk + 1][c], acc[r][c]);
          acc[r][c] = fmaf(xv.z, wa[kk + 2][c], acc[r][c]);
          acc[r][c] = fmaf(xv.w, wa[kk + 3][c], acc[r][c]);
        }
      }
    }
    const float* xk2 = xb + (size_t)(g * RG) * PITCH + ks * SLB;
#pragma unroll
    for (int kk = 0; kk < SLB; kk += 4) {
#pragma unroll
      for (int r = 0; r < RG; ++r) {
        const float4 xv = *reinterpret_cast<const float4*>(xk2 + (size_t)r * PITCH + kk);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          acc[r][c] = fmaf(xv.x, wb[kk + 0][c], acc[r][c]);
          acc[r][c] = fmaf(xv.y, wb[kk + 1][c], acc[r][c]);
          acc[r][c] = fmaf(xv.z, wb[kk + 2][c], acc[r][c]);
          acc[r][c] = fmaf(xv.w, wb[kk + 3][c], acc[r][c]);
        }
      }
    }
    const float4 s = warp_reduce_rows(acc, lane);
    *reinterpret_cast<float4*>(part + ((size_t)warp * DEC_XR + g * RG + (lane >> 2)) * NCOL + (lane & 3) * 4) = s;
  }
  __syncthreads();
  for (int o = tid; o < ngroups * RG * NCOL; o += SCAN_THREADS) {
    float s = zadd ? zadd[o] : 0.f;
#pragma unroll
    for (int wv = 0; wv < SCAN_THREADS / 32; ++wv) s += part[(size_t)wv * DEC_XR * NCOL + o];
    zout[o] = s;
  }
  __syncthreads();
}

// ---- prenet columns of a CTA: out[r][j] = xs[r][0:K] . w[0:K][j], j = 0, 1, for the staged rows ----------------
// Warp w owns rows 4w..4w+3 (no cross-warp reduction, no __syncthreads); lane l accumulates k = 128 i + 4 l .. +3
// (conflict-free float4 reads of xs).  A transposing butterfly (9 shuffles) leaves the sum of row 4w + (l >> 3),
// column (l >> 2) & 1 in lane l.  w is [K][2] in shared memory.
template <int K>
__device__ __forceinline__ float prenet_dot(const float* __restrict__ xs, const float* __restrict__ w, int lane, int warp) {
  float acc[8];   // [row][col] at 2 * row + col
#pragma unroll
  for (int v = 0; v < 8; ++v) acc[v] = 0.f;
  const float* xr = xs + (size_t)(warp * 4) * DEC_KPAD + lane * 4;
  const float* wr = w + lane * 8;
#pragma unroll 2
  for (int i = 0; i < K / 128; ++i) {
    const float4 wa = *reinterpret_cast<const float4*>(wr + i * 256);       // w[k][0..1], w[k+1][0..1]
    const float4 wb = *reinterpret_cast<const float4*>(wr + i * 256 + 4);   // w[k+2][0..1], w[k+3][0..1]
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float4 x = *reinterpret_cast<const float4*>(xr + (size_t)r * DEC_KPAD + i * 128);
      acc[2 * r] = fmaf(x.x, wa.x, acc[2 * r]); acc[2 * r + 1] = fmaf(x.x, wa.y, acc[2 * r + 1]);
      acc[2 * r] = fmaf(x.y, wa.z, acc[2 * r]); acc[2 * r + 1] = fmaf(x.y, wa.w, acc[2 * r + 1]);
      acc[2 * r] = fmaf(x.z, wb.x, acc[2 * r]); acc[2 * r + 1] = fmaf(x.z, wb.y, acc[2 * r + 1]);
      acc[2 * r] = fmaf(x.w, wb.z, acc[2 * r]); acc[2 * r + 1] = fmaf(x.w, wb.w, acc[2 * r + 1]);
    }
  }
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
  float a4[4];
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    const float send = b4 ? acc[v] : acc[v + 4];
    const float keep = b4 ? acc[v + 4] : acc[v];
    a4[v] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
  float a2[2];
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    const float send = b3 ? a4[v] : a4[v + 2];
    const float keep = b3 ? a4[v + 2] : a4[v];
    a2[v] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  float s = (b2 ? a2[1] : a2[0]) + __shfl_xor_sync(0xffffffffu, b2 ? a2[0] : a2[1], 4);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  return s;   // value index (lane >> 2) & 7 = 2 * row + col
}

// Grid barrier split in two halves (all CTAs are co-resident: cooperative launch).  dec_arrive publishes this CTA's
// stores and counts it in; work that the barrier does not order can run before dec_wait, which returns once `target`
// arrivals (a count that grows monotonically over the launch) are in.  A 2 s time-out traps instead of hanging the GPU.
__device__ __forceinline__ void dec_arrive(unsigned int* counter) {
  __syncthreads();                                   // this CTA's stores are issued
  if (threadIdx.x == 0) {
    __threadfence();                                 // ... and visible device-wide before the arrival is
    atomicAdd(counter, 1u);
  }
}
__device__ __forceinline__ void dec_wait(const unsigned int* counter, unsigned int target, int* err) {
  if (threadIdx.x == 0) {
    const long long t0 = clock64();
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (v < target && clock64() - t0 > 4000000000LL) {
        if (err) *err = 77;
        __threadfence_system();
        asm volatile("trap;");
      }
    } while (v < target);
  }
  __syncthreads();
}

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// RESUME = false: the one-shot scan of every acoustic entry point (frames 0..N-1 of every row from zero state).
// RESUME = true: one push of an acoustic stream.  Each row continues its slot from frame t0 for n steps: the carried
// state is loaded into the compact buffers (parity of frame -1) and cst, and zp0 / zp1 / p1 of the first step are
// computed from it by the same dec_matmul / prenet_dot calls that produce them from the previous frame in the one-shot
// scan, so a slot's frames get the one-shot bits.  A row past its n steps stores nothing (its state stays frozen).
template <bool RESUME>
__global__ void __launch_bounds__(SCAN_THREADS, 1) decoder_scan_kernel(const DecScanArgs a) {
  extern __shared__ __align__(16) float sm[];
  constexpr int H = vc::DEC_H, K0 = vc::PRENET + H, K1 = vc::PRENET + 2 * H;
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int B = a.B, N = a.N;
  long long tm[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  long long tq = clock64();
#define DEC_MARK(i) { const long long tn = clock64(); tm[i] += tn - tq; tq = tn; }

  float* xs = sm;                                   // [DEC_XR][DEC_KPAD] = [p2 | h0 | h1] of ONE row group at a time
  float* part = xs + DEC_XR * DEC_KPAD;             // [8][DEC_XR][16]
  float* zs = part + 8 * DEC_XR * NCOL;             // [DEC_XR][16]
  float* zp0 = zs + DEC_XR * NCOL;                  // [DEC_NG][DEC_XR][16] pre-accumulated h0_{t-1} . W0[h0 rows]
  float* zp1 = zp0 + DEC_NG * DEC_XR * NCOL;        // [DEC_NG][DEC_XR][16] pre-accumulated h1_{t-1} . W1[h1 rows]
  float* cst = zp1 + DEC_NG * DEC_XR * NCOL;        // [DEC_NG][2][DEC_XR][UPC]
  float* wcs = cst + DEC_NG * 2 * DEC_XR * UPC;     // [1024][2] (Wo . W1) columns 2c, 2c+1
  float* wp2s = wcs + 2 * H * DEC_PCOL;             // [256][2]  W2 columns 2c, 2c+1
  int4* rtab = reinterpret_cast<int4*>(wp2s + vc::PRENET * DEC_PCOL);   // RESUME: [B] row table (slot, t0, n, -)
  const int ks = tid >> 2, cgp = tid & 3;
  constexpr int SLP = vc::PRENET / NSLICE, SLH = H / NSLICE;   // 4, 8
  // register-resident weight slices, split by input segment so that each segment's product can be
  // accumulated as soon as that segment is final
  float w0p[SLP][4], w0h[SLH][4], w1p[SLP][4], w1h0[SLH][4], w1h1[SLH][4];
  {
    auto ld = [&](float (&dst)[4], const float* base, int row) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * NCOL + cgp * 4));
      dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
    };
    const float* g0 = a.w0r + (size_t)c * K0 * NCOL;
    const float* g1 = a.w1r + (size_t)c * K1 * NCOL;
#pragma unroll
    for (int i = 0; i < SLP; ++i) { ld(w0p[i], g0, ks * SLP + i); ld(w1p[i], g1, ks * SLP + i); }
#pragma unroll
    for (int i = 0; i < SLH; ++i) {
      ld(w0h[i], g0, vc::PRENET + ks * SLH + i);
      ld(w1h0[i], g1, vc::PRENET + ks * SLH + i);
      ld(w1h1[i], g1, vc::PRENET + H + ks * SLH + i);
    }
  }
  {
    const float4* gc = reinterpret_cast<const float4*>(a.wc + (size_t)c * 2 * H * DEC_PCOL);
    const float4* g2 = reinterpret_cast<const float4*>(a.wp2 + (size_t)c * vc::PRENET * DEC_PCOL);
    for (int e = tid; e < 2 * H * DEC_PCOL / 4; e += SCAN_THREADS) reinterpret_cast<float4*>(wcs)[e] = __ldg(gc + e);
    for (int e = tid; e < vc::PRENET * DEC_PCOL / 4; e += SCAN_THREADS) reinterpret_cast<float4*>(wp2s)[e] = __ldg(g2 + e);
  }
  for (int e = tid; e < DEC_NG * 2 * DEC_XR * UPC; e += SCAN_THREADS) cst[e] = 0.f;
  for (int e = tid; e < DEC_NG * 2 * DEC_XR * NCOL; e += SCAN_THREADS) zp0[e] = 0.f;   // zp0 and zp1 are adjacent
  for (int e = tid; e < DEC_XR * DEC_KPAD; e += SCAN_THREADS) xs[e] = 0.f;    // rows >= B and the t=0 state are zero
  if constexpr (RESUME)
    for (int e = tid; e < B; e += SCAN_THREADS) rtab[e] = __ldg(a.rows + e);
  __syncthreads();
  // Rows are processed in groups of DEC_XR (the staging buffer holds one group); all groups of a launch share the
  // four barriers of a frame.  With one group, h0 and p2 stay resident in xs between the phases.
  const int NG = (B + DEC_XR - 1) / DEC_XR;
  const int lastg = NG - 1, nb_last = B - lastg * DEC_XR, ng_last = (nb_last + RG - 1) / RG;
  const int prow = warp * 4 + (lane >> 3), pj = (lane >> 2) & 1, pu = DEC_PCOL * c + pj;   // prenet_dot result of this lane
  const bool pw = (lane & 3) == 0;                                                       // ... which this lane stores
  unsigned int nbar = 0;                                                                 // barriers passed so far
  // per launch row rb at local step t: the row of zc0 / zc1, the row of hout, and the (dropout row, frame) it draws
  auto zrow = [&](int rb, int t) -> size_t {
    if constexpr (RESUME) return (size_t)rtab[rb].x * a.zstride + rtab[rb].y + t;
    else return (size_t)rb * N + t;
  };
  auto hrow = [&](int rb, int t) -> size_t {
    if constexpr (RESUME) return (size_t)rb * a.hstride + t;
    else return (size_t)rb * N + t;
  };
  auto keep_at = [&](int rb, int t, int layer) -> float {
    if constexpr (RESUME) return ar_keep_scale(a.mode, a.keep, a.seed, a.subkeys, rtab[rb].x, rtab[rb].y + t, a.zstride, layer, pu);
    else return ar_keep_scale(a.mode, a.keep, a.seed, a.subkeys, a.row_base + rb, t, N, layer, pu);
  };
  auto live = [&](int rb, int t) -> bool {
    if constexpr (RESUME) return t < rtab[rb].z;
    else return true;
  };
  if constexpr (RESUME) {
    // carried state of this CTA's units -> the compact buffers at the parity of frame -1, and cst
    for (int e = tid; e < B * UPC; e += SCAN_THREADS) {
      const int rb = e / UPC, uu = e % UPC, u = c * UPC + uu, r = rb % DEC_XR;
      const float* s = a.state + (size_t)rtab[rb].x * 4 * H;
      float* cs = cst + (size_t)(rb / DEC_XR) * 2 * DEC_XR * UPC;
      a.h0[((size_t)B + rb) * H + u] = s[u];
      a.h1[((size_t)B + rb) * H + u] = s[2 * H + u];
      cs[r * UPC + uu] = s[H + u];
      cs[(DEC_XR + r) * UPC + uu] = s[3 * H + u];
    }
    dec_arrive(a.bar);
    dec_wait(a.bar, DEC_CTAS * ++nbar, a.err);        // every unit of the loaded h0 / h1 is in L2
    // zp0 = h0_{-1} . W0[h0 rows], as phase D of the previous frame computes it (with one group, h0 stays in xs)
    for (int rg = 0; rg < NG; ++rg) {
      const int r0 = rg * DEC_XR, nb = min(DEC_XR, B - r0), ngroups = (nb + RG - 1) / RG;
      dec_fetch(xs, DEC_KPAD, vc::PRENET, a.h0 + ((size_t)B + r0) * H, H, H, nb);
      __syncthreads();
      dec_matmul<SLH>(xs + vc::PRENET, w0h, ngroups, part, zp0 + rg * DEC_XR * NCOL, nullptr);
    }
  }
  for (int t = 0; t < N; ++t) {
    // ---- phase A: p1(t) = drop(relu([h0 | h1]_{t-1} . Wc + bc)) for this CTA's columns; p1(0) = 0 ----
    // (RESUME: every step takes this path from the loaded state; a row at absolute frame 0 stores p1 = 0)
    if (RESUME || t > 0) {
      for (int rg = 0; rg < NG; ++rg) {
        const int r0 = rg * DEC_XR, nb = min(DEC_XR, B - r0), ngroups = (nb + RG - 1) / RG;
        if (NG > 1) dec_fetch(xs, DEC_KPAD, vc::PRENET, a.h0 + ((size_t)((t - 1) & 1) * B + r0) * H, H, H, nb);
        dec_fetch(xs, DEC_KPAD, vc::PRENET + H, a.h1 + ((size_t)((t - 1) & 1) * B + r0) * H, H, H, nb);
        __syncthreads();
        if (warp * 4 < nb) {
          const float s = prenet_dot<2 * H>(xs + vc::PRENET, wcs, lane, warp);
          if (pw && prow < nb && live(r0 + prow, t)) {
            const float v = fmaxf(s + __ldg(a.bc + pu), 0.f);
            float* dst = a.p1 + (size_t)(r0 + prow) * vc::PRENET + pu;
            if (RESUME && rtab[r0 + prow].y + t == 0) *dst = 0.f;
            else *dst = v * keep_at(r0 + prow, t, 0);
          }
        }
        // earlier groups: their h1 leaves xs with the next fetch, so its product is taken now (the barriers inside
        // dec_matmul also order that fetch after the prenet reads)
        if (rg < lastg) dec_matmul<SLH>(xs + vc::PRENET + H, w1h1, ngroups, part, zp1 + rg * DEC_XR * NCOL, nullptr);
      }
    } else {
      for (int e = tid; e < B * DEC_PCOL; e += SCAN_THREADS) a.p1[(size_t)(e / DEC_PCOL) * vc::PRENET + DEC_PCOL * c + e % DEC_PCOL] = 0.f;
    }
    DEC_MARK(0)
    dec_arrive(a.bar);
    if (RESUME || t > 0) dec_matmul<SLH>(xs + vc::PRENET + H, w1h1, ng_last, part, zp1 + lastg * DEC_XR * NCOL, nullptr);
    for (int e = tid; e < B * 8; e += SCAN_THREADS) {   // this frame's slices of zc0 / zc1, read in phases C and D
      const int rb = e >> 3, g = (e >> 1) & 3;
      if (live(rb, t)) prefetch_l2(((e & 1) ? a.zc1 : a.zc0) + zrow(rb, t) * (4 * H) + g * H + c * UPC);
    }
    dec_wait(a.bar, DEC_CTAS * ++nbar, a.err);        // every column of p1(t) is in L2
    DEC_MARK(1)
    // ---- phase B: p2(t) = drop(relu(p1(t) . W2)) for this CTA's columns ----
    for (int rg = 0; rg < NG; ++rg) {
      const int r0 = rg * DEC_XR, nb = min(DEC_XR, B - r0);
      if (rg > 0) __syncthreads();    // the previous group's prenet reads are done
      dec_fetch(xs, DEC_KPAD, 0, a.p1 + (size_t)r0 * vc::PRENET, vc::PRENET, vc::PRENET, nb);
      __syncthreads();
      if (warp * 4 < nb) {
        const float s = prenet_dot<vc::PRENET>(xs, wp2s, lane, warp);
        if (pw && prow < nb && live(r0 + prow, t))
          a.p2[(size_t)(r0 + prow) * vc::PRENET + pu] = fmaxf(s, 0.f) * keep_at(r0 + prow, t, 1);
      }
    }
    DEC_MARK(2)
    dec_arrive(a.bar);
    dec_wait(a.bar, DEC_CTAS * ++nbar, a.err);        // every column of p2(t) is in L2
    DEC_MARK(3)
    // ---- phase C: LSTM0 = zc0[t] + p2 . W0[p2 rows] + (h0_{t-1} part) ----
    for (int rg = 0; rg < NG; ++rg) {
      const int r0 = rg * DEC_XR, nb = min(DEC_XR, B - r0), ngroups = (nb + RG - 1) / RG;
      dec_fetch(xs, DEC_KPAD, 0, a.p2 + (size_t)r0 * vc::PRENET, vc::PRENET, vc::PRENET, nb);
      __syncthreads();
      dec_matmul<SLP>(xs, w0p, ngroups, part, zs, zp0 + rg * DEC_XR * NCOL);
      if (tid < nb * UPC && live(r0 + tid / UPC, t)) {
        const int r = tid / UPC, uu = tid % UPC, rb = r0 + r;
        const float* zc = a.zc0 + zrow(rb, t) * (4 * H) + c * UPC + uu;
        float* cs = cst + (size_t)rg * 2 * DEC_XR * UPC;
        float cc = cs[r * UPC + uu];
        const float h = lstm_cell(zs, r, uu, __ldg(zc), __ldg(zc + H), __ldg(zc + 2 * H), __ldg(zc + 3 * H), cc);
        cs[r * UPC + uu] = cc;
        a.h0[((size_t)(t & 1) * B + rb) * H + c * UPC + uu] = h;
        a.hout[hrow(rb, t) * 2 * H + c * UPC + uu] = h;
        if constexpr (RESUME) {
          if (t == rtab[rb].z - 1) {   // the row's last step: carry h0, c0
            float* s = a.state + (size_t)rtab[rb].x * 4 * H + c * UPC + uu;
            s[0] = h;
            s[H] = cc;
          }
        }
      }
      if (NG > 1) __syncthreads();    // zs and xs are reused by the next group
    }
    DEC_MARK(4)
    dec_arrive(a.bar);
    dec_wait(a.bar, DEC_CTAS * ++nbar, a.err);        // h0_t is in L2
    DEC_MARK(5)
    // ---- phase D: LSTM1 = zc1[t] + p2 . W1[p2 rows] + h0_t . W1[h0 rows] + (h1_{t-1} part) ----
    const bool more = t + 1 < N;
    for (int rg = 0; rg < NG; ++rg) {
      const int r0 = rg * DEC_XR, nb = min(DEC_XR, B - r0), ngroups = (nb + RG - 1) / RG;
      if (NG > 1) dec_fetch(xs, DEC_KPAD, 0, a.p2 + (size_t)r0 * vc::PRENET, vc::PRENET, vc::PRENET, nb);
      dec_fetch(xs, DEC_KPAD, vc::PRENET, a.h0 + ((size_t)(t & 1) * B + r0) * H, H, H, nb);
      __syncthreads();
      dec_matmul2<SLP, SLH>(xs, w1p, xs + vc::PRENET, w1h0, ngroups, part, zs, zp1 + rg * DEC_XR * NCOL);
      if (tid < nb * UPC && live(r0 + tid / UPC, t)) {
        const int r = tid / UPC, uu = tid % UPC, rb = r0 + r;
        const float* zc = a.zc1 + zrow(rb, t) * (4 * H) + c * UPC + uu;
        float* cs = cst + (size_t)rg * 2 * DEC_XR * UPC;
        float cc = cs[(DEC_XR + r) * UPC + uu];
        const float h = lstm_cell(zs, r, uu, __ldg(zc), __ldg(zc + H), __ldg(zc + 2 * H), __ldg(zc + 3 * H), cc);
        cs[(DEC_XR + r) * UPC + uu] = cc;
        a.h1[((size_t)(t & 1) * B + rb) * H + c * UPC + uu] = h;
        a.hout[hrow(rb, t) * 2 * H + H + c * UPC + uu] = h;
        if constexpr (RESUME) {
          if (t == rtab[rb].z - 1) {   // the row's last step: carry h1, c1
            float* s = a.state + (size_t)rtab[rb].x * 4 * H + 2 * H + c * UPC + uu;
            s[0] = h;
            s[H] = cc;
          }
        }
      }
      // earlier groups: h0_t's product for frame t+1 while the rows are staged
      if (rg < lastg && more) dec_matmul<SLH>(xs + vc::PRENET, w0h, ngroups, part, zp0 + rg * DEC_XR * NCOL, nullptr);
      __syncthreads();
    }
    DEC_MARK(6)
    dec_arrive(a.bar);
    if (more) dec_matmul<SLH>(xs + vc::PRENET, w0h, ng_last, part, zp0 + lastg * DEC_XR * NCOL, nullptr);
    dec_wait(a.bar, DEC_CTAS * ++nbar, a.err);        // h1_t is in L2
    DEC_MARK(7)
  }
#undef DEC_MARK
  if (a.dbg && tid == 0)
    for (int i = 0; i < 8; ++i) a.dbg[(size_t)blockIdx.x * 16 + i] = tm[i];
}

// Wc[i][o] = sum_m Wo[i][m] * W1[m][o]   (1024 x 80) . (80 x 256), double accumulation; bc = bo . W1
__global__ void precompose_kernel(const float* __restrict__ wo, const float* __restrict__ bo, const float* __restrict__ w1,
                                  float* __restrict__ wc, float* __restrict__ bc) {
  const int o = threadIdx.x;            // 256
  const int i = blockIdx.x;             // 0..1024 (last block computes bc)
  double s = 0.0;
  if (i < 2 * vc::DEC_H) {
    for (int m = 0; m < vc::MEL; ++m) s += (double)wo[(size_t)i * vc::MEL + m] * (double)w1[(size_t)m * vc::PRENET + o];
    wc[(size_t)i * vc::PRENET + o] = (float)s;
  } else {
    for (int m = 0; m < vc::MEL; ++m) s += (double)bo[m] * (double)w1[(size_t)m * vc::PRENET + o];
    bc[o] = (float)s;
  }
}

// ---- teacher-forced decoder scan with zoneout (AcousticModel.__call__, model.py:146-169) ------------------
// The prenet and every input-side product are hoisted out of the recurrence (teacher forcing: the decoder input of
// frame t is the ground-truth frame t-1), so the scan only carries  h0s.W0[h0 rows],  h0n.W1[h0 rows]  and
// h1s.W1[h1 rows].  *n = the cores' new state (what the decoder outputs), *s = the state after zoneout
// (state = mask ? previous : new, model.py:157-159).  One grid barrier per frame: iteration s runs LSTM0 of frame s
// and LSTM1 of frame s-1 -- both only need values published in iteration s-1.
struct TfScanArgs {
  const float* zc0;      // [B][N][2048]  [cond, p2] . W0[0:768] + b0
  const float* zc1;      // [B][N][2048]  [cond, p2] . W1[0:768] + b1
  const float* w0r;      // [128][768][16]   rows 512..1279 of lstm0 ([p2, h0]); only the h0 rows are used here
  const float* w1r;      // [128][1280][16]  rows 512..1791 of lstm1 ([p2, h0, h1]); h0 and h1 rows used
  const uint8_t* zone;   // [B][N][4][512] (h0, c0, h1, c1; 1 = keep the previous state) or null
  uint64_t seed;
  int mode;              // VTTS_DROPOUT_OFF / MASK / SEED / REFERENCE
  uint2 zkey[4];         // REFERENCE: sub-keys of the four zoneout draws (state order h0, c0, h1, c1)
  float* h0s;            // [2][B][512] zoned hidden state of layer 0, double buffered by frame parity
  float* h1s;            // [2][B][512]
  float* hout;           // [B][N][1024]  decoder outputs [h0n | h1n]
  int B, N;
  int row_base;
  int B_call;            // rows of the whole call (the REFERENCE draws span the call's batch, not this launch's rows)
};

constexpr int TF_PITCH = 3 * vc::DEC_H + 4;    // [h0s | h0n | h1s] + pad

// true = keep the previous state.  SEED mode: Bernoulli(0.1) from the same threefry stream as the prenet masks,
// counter word 1 offset past the prenet's 2*256 entries.  REFERENCE mode: element (b, t, unit) of the reference's
// bernoulli(zkey[which], 0.1, [B,N,512]) draw over the call's B rows, with jax's float32 compare.
__device__ __forceinline__ bool zone_keep(int mode, const uint8_t* zone, uint64_t seed, uint2 rkey, int b, int t, int B, int N, int which,
                                          int unit) {
  if (mode == VTTS_DROPOUT_OFF) return false;
  if (mode == VTTS_DROPOUT_MASK) return zone[(((size_t)b * N + t) * 4 + which) * vc::DEC_H + unit] != 0;
  const uint32_t w = stream_word(mode, seed, b, t, (uint32_t)(2 * vc::PRENET + which * vc::DEC_H + unit), rkey,
                                 ((uint32_t)b * N + t) * vc::DEC_H + unit, (uint32_t)B * N * vc::DEC_H);
  if (mode == VTTS_DROPOUT_REFERENCE) return __uint_as_float((w >> 9) | 0x3F800000u) - 1.f < 0.1f;
  return w < 429496730u;   // 0.1 * 2^32
}

__global__ void __launch_bounds__(SCAN_THREADS, 1) decoder_tf_scan_kernel(const TfScanArgs a) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) float sm[];
  constexpr int H = vc::DEC_H, K0 = vc::PRENET + H, K1 = vc::PRENET + 2 * H, SLH = H / NSLICE;   // 8
  const int c = blockIdx.x, tid = threadIdx.x;
  const int B = a.B, N = a.N;
  float* xs = sm;                                   // [DEC_XR][TF_PITCH]
  float* part = xs + DEC_XR * TF_PITCH;             // [8][DEC_XR][16]
  float* zs = part + 8 * DEC_XR * NCOL;             // [DEC_XR][16]
  float* cst = zs + DEC_XR * NCOL;                  // [2][DEC_XR][UPC] zoned cell states of the CTA's units
  const int ks = tid >> 2, cgp = tid & 3;
  float w0h[SLH][4], w1h0[SLH][4], w1h1[SLH][4];
  {
    auto ld = [&](float (&dst)[4], const float* base, int row) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * NCOL + cgp * 4));
      dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
    };
    const float* g0 = a.w0r + (size_t)c * K0 * NCOL;
    const float* g1 = a.w1r + (size_t)c * K1 * NCOL;
#pragma unroll
    for (int i = 0; i < SLH; ++i) {
      ld(w0h[i], g0, vc::PRENET + ks * SLH + i);
      ld(w1h0[i], g1, vc::PRENET + ks * SLH + i);
      ld(w1h1[i], g1, vc::PRENET + H + ks * SLH + i);
    }
  }
  for (int e = tid; e < 2 * DEC_XR * UPC; e += SCAN_THREADS) cst[e] = 0.f;
  for (int e = tid; e < DEC_XR * TF_PITCH; e += SCAN_THREADS) xs[e] = 0.f;
  __syncthreads();
  const int ngroups = (B + RG - 1) / RG;
  for (int s = 0; s <= N; ++s) {
    // values published in iteration s-1: h0s_{s-1}, h0n_{s-1} (LSTM0 of frame s-1) and h1s_{s-2} (LSTM1 of frame s-2)
    // three copy groups in flight: LSTM0 of frame s only needs the first one, the operands of LSTM1 (frame s-1) keep
    // arriving while its product runs
    if (s >= 1) {
      dec_fetch_async(xs, TF_PITCH, 0, a.h0s + (size_t)((s - 1) & 1) * B * H, H, H, B);
      dec_fetch_async(xs, TF_PITCH, H, a.hout + (size_t)(s - 1) * 2 * H, H, N * 2 * H, B);
    } else {
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (s >= 2) dec_fetch_async(xs, TF_PITCH, 2 * H, a.h1s + (size_t)(s & 1) * B * H, H, H, B);
    else asm volatile("cp.async.commit_group;" ::: "memory");
    cp_async_wait<2>();
    __syncthreads();
    if (s < N) {
      // ---- LSTM0 of frame s: z = zc0[s] + h0s_{s-1} . W0[h0 rows] ----
      dec_matmul<SLH, TF_PITCH>(xs, w0h, ngroups, part, zs, nullptr);
      if (tid < B * UPC) {
        const int r = tid / UPC, uu = tid % UPC, u = c * UPC + uu;
        const float* zc = a.zc0 + ((size_t)r * N + s) * (4 * H) + u;
        const float c_prev = cst[r * UPC + uu];
        float cc = c_prev;
        const float h = lstm_cell(zs, r, uu, __ldg(zc), __ldg(zc + H), __ldg(zc + 2 * H), __ldg(zc + 3 * H), cc);
        const bool kh = zone_keep(a.mode, a.zone, a.seed, a.zkey[0], a.row_base + r, s, a.B_call, N, 0, u);
        const bool kc = zone_keep(a.mode, a.zone, a.seed, a.zkey[1], a.row_base + r, s, a.B_call, N, 1, u);
        a.hout[((size_t)r * N + s) * 2 * H + u] = h;
        a.h0s[((size_t)(s & 1) * B + r) * H + u] = kh ? xs[(size_t)r * TF_PITCH + u] : h;
        cst[r * UPC + uu] = kc ? c_prev : cc;
      }
    }
    cp_async_wait<0>();
    if (s >= 1) {
      // ---- LSTM1 of frame s-1: z = zc1[s-1] + h0n_{s-1} . W1[h0 rows] + h1s_{s-2} . W1[h1 rows] ----
      const int t = s - 1;
      __syncthreads();    // zs is reused; every thread's copies of the LSTM1 operands have landed
      dec_matmul2<SLH, SLH, TF_PITCH>(xs + H, w1h0, xs + 2 * H, w1h1, ngroups, part, zs, nullptr);
      if (tid < B * UPC) {
        const int r = tid / UPC, uu = tid % UPC, u = c * UPC + uu;
        const float* zc = a.zc1 + ((size_t)r * N + t) * (4 * H) + u;
        const float c_prev = cst[(DEC_XR + r) * UPC + uu];
        float cc = c_prev;
        const float h = lstm_cell(zs, r, uu, __ldg(zc), __ldg(zc + H), __ldg(zc + 2 * H), __ldg(zc + 3 * H), cc);
        const bool kh = zone_keep(a.mode, a.zone, a.seed, a.zkey[2], a.row_base + r, t, a.B_call, N, 2, u);
        const bool kc = zone_keep(a.mode, a.zone, a.seed, a.zkey[3], a.row_base + r, t, a.B_call, N, 3, u);
        a.hout[((size_t)r * N + t) * 2 * H + H + u] = h;
        a.h1s[((size_t)(t & 1) * B + r) * H + u] = kh ? xs[(size_t)r * TF_PITCH + 2 * H + u] : h;
        cst[(DEC_XR + r) * UPC + uu] = kc ? c_prev : cc;
      }
    }
    __syncthreads();
    grid.sync();
  }
}

// out[row][c] (row stride out_ld) = relu(x[row][c]) * keep_scale  -- the two prenet dropouts applied to whole sequences
// (rkey: the REFERENCE sub-key of this layer's draw)
__global__ void prenet_act_kernel(const float* __restrict__ x, const uint8_t* __restrict__ keep, uint64_t seed, int mode, uint2 rkey,
                                  int layer, int B, int N, float* __restrict__ out, int out_ld) {
  const size_t total = (size_t)B * N * vc::PRENET;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int u = (int)(i % vc::PRENET);
    const size_t row = i / vc::PRENET;
    const int b = (int)(row / N), t = (int)(row % N);
    out[row * out_ld + u] = fmaxf(x[i], 0.f) * tf_keep_scale(mode, keep, seed, rkey, b, t, B, N, layer, u);
  }
}

// Test hook kernels: the masks REFERENCE mode applies, through the draw functions of the scans above.
// [N][2][256] of the autoregressive scan (row 0; every row shares them)
__global__ void ref_ar_masks_kernel(const uint2* __restrict__ subkeys, int N, uint8_t* __restrict__ out) {
  const size_t total = (size_t)N * 2 * vc::PRENET;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int u = (int)(i % vc::PRENET), l = (int)((i / vc::PRENET) % 2), t = (int)(i / (2 * vc::PRENET));
    out[i] = ar_keep_scale(VTTS_DROPOUT_REFERENCE, nullptr, 0, subkeys, 0, t, N, l, u) != 0.f;
  }
}
// teacher-forced pass: keep [B][N][2][256], zone [B][N][4][512]
__global__ void ref_tf_masks_kernel(uint2 k0, uint2 k1, uint2 z0, uint2 z1, uint2 z2, uint2 z3, int B, int N, uint8_t* __restrict__ keep,
                                    uint8_t* __restrict__ zone) {
  const size_t nk = (size_t)B * N * 2 * vc::PRENET, nz = (size_t)B * N * 4 * vc::DEC_H;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nk + nz; i += (size_t)gridDim.x * blockDim.x) {
    if (i < nk) {
      const int u = (int)(i % vc::PRENET), l = (int)((i / vc::PRENET) % 2);
      const size_t row = i / (2 * vc::PRENET);
      const int b = (int)(row / N), t = (int)(row % N);
      keep[i] = tf_keep_scale(VTTS_DROPOUT_REFERENCE, nullptr, 0, l ? k1 : k0, b, t, B, N, l, u) != 0.f;
    } else {
      const size_t j = i - nk;
      const int u = (int)(j % vc::DEC_H), w = (int)((j / vc::DEC_H) % 4);
      const size_t row = j / (4 * vc::DEC_H);
      const int b = (int)(row / N), t = (int)(row % N);
      const uint2 zk = w == 0 ? z0 : (w == 1 ? z1 : (w == 2 ? z2 : z3));
      zone[j] = zone_keep(VTTS_DROPOUT_REFERENCE, nullptr, 0, zk, b, t, B, N, w, u);
    }
  }
}

constexpr size_t tf_scan_smem() { return ((size_t)DEC_XR * TF_PITCH + 8 * DEC_XR * NCOL + DEC_XR * NCOL + 2 * DEC_XR * UPC) * 4; }

constexpr size_t enc_scan_smem() {
  return ((size_t)32 * (vc::ENC_D + 4) + 8 * DEC_XR * NCOL + DEC_XR * NCOL + MAX_ROWS * UPC) * 4;
}
constexpr size_t dec_scan_smem() {
  return ((size_t)DEC_XR * DEC_KPAD + 8 * DEC_XR * NCOL + DEC_XR * NCOL + DEC_NG * (2 * DEC_XR * NCOL + 2 * DEC_XR * UPC) +
          (2 * vc::DEC_H + vc::PRENET) * DEC_PCOL) * 4;
}
static_assert(dec_scan_smem() <= 227 * 1024, "decoder scan shared memory exceeds the 227 KB of an sm_90 CTA");
// the RESUME instantiation adds its row table after the prenet weights
constexpr size_t dec_resume_smem() { return dec_scan_smem() + (size_t)MAX_ROWS * sizeof(int4); }
static_assert(dec_resume_smem() <= 227 * 1024, "resumable decoder scan shared memory exceeds the 227 KB of an sm_90 CTA");

// Slot layout shared by the acoustic and the duration model: the TokenEncoder's derived tensors and packed convs
// come first in both, so that run_token_encoder reads either slot.
enum { D_ENC_BNINV0, D_ENC_BNINV1, D_ENC_BNINV2,
       D_ENC_WHR,     // [2][64][256][16]
       D_ENC_COUNT };
enum { PK_ENC_CONV0, PK_ENC_CONV1, PK_ENC_CONV2, PK_ENC_LSTM_F, PK_ENC_LSTM_B, PK_ENC_COUNT };

// derived tensors of the acoustic model (ctx->ac.d)
enum {
  D_POST_BNINV0 = D_ENC_COUNT, D_POST_BNINV1, D_POST_BNINV2, D_POST_BNINV3,
  D_DEC_W0R,     // [128][768][16]
  D_DEC_W1R,     // [128][1280][16]
  D_DEC_WC,      // [128][1024][2]  (Wo . W1) columns 2c, 2c+1 of decoder-scan CTA c
  D_DEC_WCFULL,  // [1024][256] scratch
  D_DEC_BC,      // [256]
  D_DEC_WP2,     // [128][256][2]   prenet fc2 columns 2c, 2c+1 of decoder-scan CTA c
  D_ZERO,        // [2048] zeros: bias of the bias-free prenet linears (model.py:88-89) on the generic conv path
  D_COUNT
};

// packing table of the acoustic model (ctx->ac.tiles).  The problems of one multi-problem launch are consecutive
// entries: the two decoder LSTMs, and the teacher-forced pass's [cond | p2] rows 0..767 of both
enum { PK_DEC_L0 = PK_ENC_COUNT, PK_DEC_L1, PK_POST0, PK_PROJ = PK_POST0 + 5, PK_TF_L0, PK_TF_L1, PK_PRE1, PK_PRE2, PK_COUNT };

}  // namespace

// TokenEncoder.__call__ (model.py:26-47, is_training=False): embed -> 3 x [conv k3, BN(eval), relu] -> BiLSTM.
// The acoustic model and the duration model instantiate it with the same dimensions (config.py:11-17) and their
// slots share its layout (aci::EMBED .. aci::ENC_LSTM_B_B, D_ENC_*, PK_ENC_*), so one implementation serves both.
static void encoder_tables(const ModelWeights& m, std::vector<size_t>& dn, std::vector<PackSpec>& pk) {
  const auto& T = m.t;
  for (int i = 0; i < 3; ++i) {
    dn[D_ENC_BNINV0 + i] = 256;
    pk[PK_ENC_CONV0 + i] = {T[aci::ENC_CONV(i, 0)], 3, 256, 256};
  }
  dn[D_ENC_WHR] = (size_t)2 * 64 * 256 * 16;
  pk[PK_ENC_LSTM_F] = {T[aci::ENC_LSTM_F_W], 1, 256, 1024};
  pk[PK_ENC_LSTM_B] = {T[aci::ENC_LSTM_B_W], 1, 256, 1024};
}

static void encoder_derive(const ModelWeights& m) {
  const auto& T = m.t;
  for (int i = 0; i < 3; ++i) vtts_bn_inv(T[aci::ENC_CONV(i, 2)], T[aci::ENC_CONV(i, 5)], m.d[D_ENC_BNINV0 + i], 256);
  // recurrent weights: rows 256..511 of w[512][1024]
  repack_cols_kernel<<<256, 256>>>(T[aci::ENC_LSTM_F_W], 1024, 256, 256, m.d[D_ENC_WHR], 64, 16, UPC, 256);
  repack_cols_kernel<<<256, 256>>>(T[aci::ENC_LSTM_B_W], 1024, 256, 256, m.d[D_ENC_WHR] + (size_t)64 * 256 * 16, 64, 16, UPC, 256);
}

// ConvProb of a "same"-padded dilation-1 conv of kernel size k (k = 1: a GEMM over rows); the other fields are zero
static ConvProb conv_prob(const float* x, const float* w, const float* bias, float* out, int k = 1) {
  ConvProb p;
  memset(&p, 0, sizeof(p));
  p.x0 = x; p.w = w; p.bias = bias; p.out = out;
  p.k = k; p.dil = 1; p.in_off = -(k - 1) / 2; p.out_stride = 1;
  return p;
}

// nprob problems of one shape over B sequences of T rows (rows past len[b] are skipped when len is given), through
// the shared dispatch: tensor-core path in BF16X3 mode (packed tiles `wpk`), FMA path in FP32 mode
static int run_convs(vtts_ctx* ctx, const ConvProb* p, int nprob, int Cin, int Cout, int B, int T, const int32_t* len,
                     int post_act, void* const* wpk, cudaStream_t st) {
  ConvLaunch L;
  memset(&L, 0, sizeof(L));
  for (int i = 0; i < nprob; ++i) L.p[i] = p[i];
  L.nprob = nprob; L.Cin = Cin; L.Cout = Cout; L.B = B; L.T_rows = T; L.rows_out = T;
  L.len = len; L.len_mul = 1; L.pre_mode = 0; L.pre_slope = 1.f; L.post_act = post_act;
  return vtts_conv_dispatch(ctx, L, wpk, st);
}

struct EncBufs { float *e0, *e1, *zx, *enc; };

static void carve_encoder(Arena& ar, size_t BL, EncBufs& e) {
  e.e0 = ar.take<float>(BL * 256);
  e.e1 = ar.take<float>(BL * 256);
  e.zx = ar.take<float>(2 * BL * 1024);
  e.enc = ar.take<float>(BL * 512);
}

static int run_token_encoder(vtts_ctx* ctx, const ModelWeights& m, const int32_t* tokens, const int32_t* lengths, int B, int L,
                             const EncBufs& e, cudaStream_t st) {
  const auto& T = m.t;
  const size_t BL = (size_t)B * L;
  embed_kernel<<<(unsigned)((BL + 3) / 4), 256, 0, st>>>(tokens, T[aci::EMBED], e.e0, (int)BL);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  float* cur = e.e0;
  float* nxt = e.e1;
  for (int i = 0; i < 3; ++i) {
    ConvProb p = conv_prob(cur, T[aci::ENC_CONV(i, 0)], T[aci::ENC_CONV(i, 1)], nxt, 3);
    p.bn_mean = T[aci::ENC_CONV(i, 4)]; p.bn_inv = m.d[D_ENC_BNINV0 + i]; p.bn_off = T[aci::ENC_CONV(i, 3)];
    int rc = run_convs(ctx, &p, 1, 256, 256, B, L, lengths, 2, m.tiles(PK_ENC_CONV0 + i), st);
    if (rc) return rc;
    float* tmp = cur; cur = nxt; nxt = tmp;
  }
  // rows past len[b] of `cur` were never written: the scans mask them, but the hoisted GEMM reads them
  // -> harmless garbage confined to rows that are never consumed (k=1 GEMM has no row mixing).
  // ---- hoisted input projections of the two LSTMs: zx[dir] = x . W[0:256] + b ----
  const ConvProb hp[2] = {conv_prob(cur, T[aci::ENC_LSTM_F_W], T[aci::ENC_LSTM_F_B], e.zx),
                          conv_prob(cur, T[aci::ENC_LSTM_B_W], T[aci::ENC_LSTM_B_B], e.zx + BL * 1024)};
  int rc = run_convs(ctx, hp, 2, 256, 1024, 1, (int)BL, nullptr, 0, m.tiles(PK_ENC_LSTM_F), st);
  if (rc) return rc;
  // ---- BiLSTM scan (forward core + ResetCore'd backward core) ----
  EncScanArgs ea;
  ea.zx = e.zx; ea.whr = m.d[D_ENC_WHR]; ea.lengths = lengths; ea.out = e.enc; ea.B = B; ea.L = L;
  void* args[] = {&ea};
  VTTS_CUDA(cudaLaunchCooperativeKernel((void*)enc_scan_kernel, dim3(SCAN_CTAS), dim3(SCAN_THREADS), args, enc_scan_smem(), st));
  ctx->launches++;
  return VTTS_OK;
}

int vtts_acoustic_prepare(vtts_ctx* ctx) {
  ModelWeights& m = ctx->ac;
  const auto& T = m.t;
  std::vector<size_t> dn(D_COUNT);
  std::vector<PackSpec> pk(PK_COUNT);
  encoder_tables(m, dn, pk);
  for (int i = 0; i < 4; ++i) dn[D_POST_BNINV0 + i] = 512;
  dn[D_DEC_W0R] = (size_t)128 * 768 * 16;
  dn[D_DEC_W1R] = (size_t)128 * 1280 * 16;
  dn[D_DEC_WC] = (size_t)DEC_CTAS * 1024 * DEC_PCOL;
  dn[D_DEC_WCFULL] = (size_t)1024 * 256;
  dn[D_DEC_BC] = 256;
  dn[D_DEC_WP2] = (size_t)DEC_CTAS * 256 * DEC_PCOL;
  dn[D_ZERO] = 2048;
  pk[PK_DEC_L0] = {T[aci::DEC_L0_W], 1, 512, 2048};
  pk[PK_DEC_L1] = {T[aci::DEC_L1_W], 1, 512, 2048};
  for (int i = 0; i < 5; ++i) pk[PK_POST0 + i] = {T[aci::POST_CONV(i, 0)], 5, i == 0 ? 80 : 512, i == 4 ? 80 : 512};
  pk[PK_PROJ] = {T[aci::PROJ_W], 1, 1024, 80};
  pk[PK_TF_L0] = {T[aci::DEC_L0_W], 1, 768, 2048};
  pk[PK_TF_L1] = {T[aci::DEC_L1_W], 1, 768, 2048};
  pk[PK_PRE1] = {T[aci::PRE1_W], 1, 80, 256};
  pk[PK_PRE2] = {T[aci::PRE2_W], 1, 256, 256};
  int rc = vtts_alloc_tensors(ctx, dn, &m.derived, m.d);   // zero-filled: D_ZERO needs no further work
  if (rc) return rc;
  encoder_derive(m);
  for (int i = 0; i < 4; ++i) vtts_bn_inv(T[aci::POST_CONV(i, 2)], T[aci::POST_CONV(i, 5)], m.d[D_POST_BNINV0 + i], 512);
  // decoder: rows after the 512 cond rows
  repack_cols_kernel<<<512, 256>>>(T[aci::DEC_L0_W], 2048, 512, 768, m.d[D_DEC_W0R], 128, 16, UPC, 512);
  repack_cols_kernel<<<512, 256>>>(T[aci::DEC_L1_W], 2048, 512, 1280, m.d[D_DEC_W1R], 128, 16, UPC, 512);
  precompose_kernel<<<2 * vc::DEC_H + 1, 256>>>(T[aci::PROJ_W], T[aci::PROJ_B], T[aci::PRE1_W], m.d[D_DEC_WCFULL], m.d[D_DEC_BC]);
  repack_cols_kernel<<<256, 256>>>(m.d[D_DEC_WCFULL], 256, 0, 1024, m.d[D_DEC_WC], DEC_CTAS, DEC_PCOL, DEC_PCOL, 0);
  repack_cols_kernel<<<64, 256>>>(T[aci::PRE2_W], 256, 0, 256, m.d[D_DEC_WP2], DEC_CTAS, DEC_PCOL, DEC_PCOL, 0);
  VTTS_CUDA(cudaGetLastError());
  rc = vtts_pack_convs(ctx, m, pk);
  if (rc) return rc;
  VTTS_CUDA(cudaDeviceSynchronize());
  VTTS_CUDA(cudaFuncSetAttribute(enc_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)enc_scan_smem()));
  VTTS_CUDA(cudaFuncSetAttribute(decoder_scan_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dec_scan_smem()));
  VTTS_CUDA(cudaFuncSetAttribute(decoder_scan_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dec_resume_smem()));
  VTTS_CUDA(cudaFuncSetAttribute(decoder_tf_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tf_scan_smem()));
  return VTTS_OK;
}

// Gaussian upsampling of the encoder output to N frames: columns 0..511 of `out` (row stride out_ld)
static int run_upsample(vtts_ctx* ctx, const float* enc, const float* dur, const int32_t* lengths, const int32_t* n_frames,
                        int B, int L, int N, float* out, int out_ld, cudaStream_t st) {
  dim3 grid((N + UP_F - 1) / UP_F, B);
  size_t smem = (size_t)(L + UP_F * L) * sizeof(float);
  if (smem > 200 * 1024) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic: L=%d too long for the upsample kernel", L);
  if (smem > 48 * 1024) VTTS_CUDA(cudaFuncSetAttribute(upsample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  upsample_kernel<<<grid, 256, smem, st>>>(enc, dur, lengths, n_frames, L, N, out, out_ld);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// Output projection of every frame in one GEMM, melpre = [h0 | h1] . Wo + bo (model.py:135; rows past n_frames[b] stay 0),
// copied to mel1 if given; sub-stage mark `proj_mark` (if >= 0); then AcousticModel.postnet (model.py:113-121,
// is_training=False) + the residual add (:143-144 / :169): mel = melpre + conv5(tanh(bn(conv5(...)))).
// q0/q1 are [B*N][512] scratch.
int vtts_acoustic_project(vtts_ctx* ctx, const float* hout, const int32_t* len, int B, int T, float* melpre, cudaStream_t st) {
  const ModelWeights& m = ctx->ac;
  const ConvProb pp = conv_prob(hout, m.t[aci::PROJ_W], m.t[aci::PROJ_B], melpre);
  return run_convs(ctx, &pp, 1, 1024, 80, B, T, len, 0, m.tiles(PK_PROJ), st);
}

int vtts_acoustic_postnet(vtts_ctx* ctx, const float* melpre, const int32_t* len, int B, int T, float* q0, float* q1, float* mel,
                          cudaStream_t st) {
  const ModelWeights& m = ctx->ac;
  const auto& W = m.t;
  const float* pin = melpre;
  float* pout = q0;
  for (int i = 0; i < 5; ++i) {
    ConvProb p = conv_prob(pin, W[aci::POST_CONV(i, 0)], W[aci::POST_CONV(i, 1)], i < 4 ? pout : mel, 5);
    if (i < 4) { p.bn_mean = W[aci::POST_CONV(i, 4)]; p.bn_inv = m.d[D_POST_BNINV0 + i]; p.bn_off = W[aci::POST_CONV(i, 3)]; }
    else p.resid = melpre;
    const int rc = run_convs(ctx, &p, 1, i == 0 ? 80 : 512, i < 4 ? 512 : 80, B, T, len, i < 4 ? 1 : 0, m.tiles(PK_POST0 + i), st);
    if (rc) return rc;
    pin = pout;
    pout = (pout == q0) ? q1 : q0;
  }
  return VTTS_OK;
}

static int run_projection_postnet(vtts_ctx* ctx, const float* hout, const int32_t* n_frames, int B, int N, float* melpre,
                                  float* q0, float* q1, float* mel1, int proj_mark, float* mel, cudaStream_t st) {
  int rc = vtts_acoustic_project(ctx, hout, n_frames, B, N, melpre, st);
  if (rc) return rc;
  if (mel1) VTTS_CUDA(cudaMemcpyAsync(mel1, melpre, (size_t)B * N * 80 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (proj_mark >= 0) ctx->sub_mark(proj_mark, st);
  return vtts_acoustic_postnet(ctx, melpre, n_frames, B, N, q0, q1, mel, st);
}

namespace {
// Workspace of one pass.  carve() lays it out the same way for sizing (*_ws_bytes) and for the run.
struct AcBufs {
  EncBufs e;
  float *cond, *zc0, *zc1, *melpre, *q0, *q1, *p1, *p2, *hout, *h0, *h1;
  unsigned int* dec_bar;
  uint2* subkeys;   // [N][2] REFERENCE sub-keys
};
struct TfBufs {
  EncBufs e;
  float *xin, *pa, *pb, *zc0, *zc1, *hout, *melpre, *q0, *q1, *h0s, *h1s;
};
struct DuBufs {
  EncBufs e;
  float* y;
};
constexpr int XW = vc::ENC_OUT + vc::PRENET;   // 768: teacher-forced decoder input [cond | prenet(mel)]

void carve(Arena& ar, int B, int L, int N, AcBufs& w) {
  const size_t BN = (size_t)B * N;
  carve_encoder(ar, (size_t)B * L, w.e);
  w.cond = ar.take<float>(BN * 512);
  w.zc0 = ar.take<float>(BN * 2048);
  w.zc1 = ar.take<float>(BN * 2048);
  w.melpre = ar.take<float>(BN * 80);
  w.q0 = ar.take<float>(BN * 512);
  w.q1 = ar.take<float>(BN * 512);
  w.p1 = ar.take<float>((size_t)B * 256);
  w.p2 = ar.take<float>((size_t)B * 256);
  w.hout = ar.take<float>(BN * 1024);
  w.h0 = ar.take<float>((size_t)2 * MAX_ROWS * 512);
  w.h1 = ar.take<float>((size_t)2 * MAX_ROWS * 512);
  w.dec_bar = ar.take<unsigned int>(64);
  w.subkeys = ar.take<uint2>((size_t)2 * N);
}
void carve(Arena& ar, int B, int L, int N, TfBufs& w) {
  const size_t BN = (size_t)B * N;
  carve_encoder(ar, (size_t)B * L, w.e);
  w.xin = ar.take<float>(BN * XW);
  w.pa = ar.take<float>(BN * 256);
  w.pb = ar.take<float>(BN * 256);
  w.zc0 = ar.take<float>(BN * 2048);
  w.zc1 = ar.take<float>(BN * 2048);
  w.hout = ar.take<float>(BN * 1024);
  w.melpre = ar.take<float>(BN * 80);
  w.q0 = ar.take<float>(BN * 512);
  w.q1 = ar.take<float>(BN * 512);
  w.h0s = ar.take<float>((size_t)2 * DEC_XR * 512);
  w.h1s = ar.take<float>((size_t)2 * DEC_XR * 512);
}
void carve(Arena& ar, int B, int L, int, DuBufs& w) {
  carve_encoder(ar, (size_t)B * L, w.e);
  w.y = ar.take<float>((size_t)B * L * 256);
}
template <class Bufs>
size_t ws_bytes(int B, int L, int N) {
  Arena ar(nullptr, 0, true);
  Bufs w;
  carve(ar, B, L, N, w);
  return ar.off + 256;
}
template <class Bufs>
Bufs carve_ws(vtts_ctx* ctx, int B, int L, int N) {
  Arena ar(ctx->ws, ctx->ws_bytes, false);
  Bufs w;
  carve(ar, B, L, N, w);
  return w;
}
}  // namespace

size_t vtts_acoustic_ws_bytes(int B, int L, int N) { return ws_bytes<AcBufs>(B, L, N); }
size_t vtts_acoustic_teacher_ws_bytes(int B, int L, int N) { return ws_bytes<TfBufs>(B, L, N); }
size_t vtts_duration_ws_bytes(int B, int L) { return ws_bytes<DuBufs>(B, L, 0); }

// TokenEncoder -> upsample -> hoisted cond projections zc0 / zc1 of the decoder LSTMs (sub-stage marks 0..3)
static int run_acoustic_front(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur, const int32_t* n_frames,
                              int B, int L, int N, const AcBufs& w, cudaStream_t st) {
  const ModelWeights& m = ctx->ac;
  const auto& T = m.t;
  const size_t BN = (size_t)B * N;
  VTTS_CUDA(cudaMemsetAsync(w.cond, 0, BN * 512 * sizeof(float), st));
  ctx->sub_mark(0, st);
  int rc = run_token_encoder(ctx, m, tokens, lengths, B, L, w.e, st);
  if (rc) return rc;
  ctx->sub_mark(1, st);
  rc = run_upsample(ctx, w.e.enc, dur, lengths, n_frames, B, L, N, w.cond, vc::ENC_OUT, st);
  if (rc) return rc;
  ctx->sub_mark(2, st);
  const ConvProb hp[2] = {conv_prob(w.cond, T[aci::DEC_L0_W], T[aci::DEC_L0_B], w.zc0), conv_prob(w.cond, T[aci::DEC_L1_W], T[aci::DEC_L1_B], w.zc1)};
  rc = run_convs(ctx, hp, 2, 512, 2048, 1, (int)BN, nullptr, 0, m.tiles(PK_DEC_L0), st);
  if (rc) return rc;
  ctx->sub_mark(3, st);
  return VTTS_OK;
}

int vtts_acoustic_front(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur, const int32_t* n_frames, int B,
                        int L, int N, const float** zc0, const float** zc1, cudaStream_t st) {
  if (!ctx->ac.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "acoustic weights not loaded");
  if (B < 1 || L < 1 || N < 1 || B > MAX_ROWS) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic: B=%d L=%d N=%d", B, L, N);
  const AcBufs w = carve_ws<AcBufs>(ctx, B, L, N);
  *zc0 = w.zc0;
  *zc1 = w.zc1;
  return run_acoustic_front(ctx, tokens, lengths, dur, n_frames, B, L, N, w, st);
}

int vtts_ref_subkeys(vtts_ctx* ctx, uint64_t seed, int n, uint2* out, cudaStream_t st) {
  ref_subkey_chain_kernel<<<1, 32, 0, st>>>(seed, n, out);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

int vtts_decoder_scan_resume(vtts_ctx* ctx, const DecResume& r, cudaStream_t st) {
  if (r.B < 1 || r.B > MAX_ROWS || r.nmax < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "decoder_scan_resume: B=%d nmax=%d", r.B, r.nmax);
  if (ctx->sm_count < DEC_CTAS) return ctx->fail(VTTS_ERR_NO_DEVICE, "scan kernels need %d SMs, device has %d", DEC_CTAS, ctx->sm_count);
  const ModelWeights& m = ctx->ac;
  const auto& D = m.d;
  DecScanArgs da;
  memset(&da, 0, sizeof(da));
  da.zc0 = r.zc0; da.zc1 = r.zc1;
  da.w0r = D[D_DEC_W0R]; da.w1r = D[D_DEC_W1R]; da.wc = D[D_DEC_WC]; da.bc = D[D_DEC_BC]; da.wp2 = D[D_DEC_WP2];
  da.keep = r.keep; da.subkeys = r.subkeys; da.seed = r.seed; da.mode = r.mode;
  da.p1 = r.p1; da.p2 = r.p2; da.h0 = r.h0; da.h1 = r.h1; da.hout = r.hout;
  da.bar = r.bar; da.err = ctx->d_err;
  da.B = r.B; da.N = r.nmax; da.row_base = 0;
  da.rows = r.rows; da.state = r.state; da.zstride = r.zstride; da.hstride = r.hstride;
  VTTS_CUDA(cudaMemsetAsync(r.bar, 0, sizeof(unsigned int), st));
  void* args[] = {&da};
  VTTS_CUDA(cudaLaunchCooperativeKernel((void*)decoder_scan_kernel<true>, dim3(DEC_CTAS), dim3(SCAN_THREADS), args, dec_resume_smem(), st));
  ctx->launches++;
  return VTTS_OK;
}

int vtts_acoustic_max_tokens() { return (200 * 1024) / (int)((1 + UP_F) * sizeof(float)); }

int vtts_acoustic_run(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur,
                      const int32_t* n_frames, const uint8_t* keep, int mode, uint64_t seed, int B, int L, int N,
                      float* mel, cudaStream_t st) {
  if (!ctx->ac.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "acoustic weights not loaded");
  if (B < 1 || L < 1 || N < 1 || B > MAX_ROWS)
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic: B=%d L=%d N=%d (1 <= B <= %d rows per call; the host layer chunks larger batches)", B, L, N, MAX_ROWS);
  if (mode < VTTS_DROPOUT_OFF || mode > VTTS_DROPOUT_REFERENCE) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic: dropout_mode %d", mode);
  if (mode == VTTS_DROPOUT_MASK && !keep) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic: dropout_mode MASK needs keep_mask");
  if (ctx->sm_count < DEC_CTAS) return ctx->fail(VTTS_ERR_NO_DEVICE, "scan kernels need %d SMs, device has %d", DEC_CTAS, ctx->sm_count);
  const AcBufs w = carve_ws<AcBufs>(ctx, B, L, N);
  const size_t BL = (size_t)B * L, BN = (size_t)B * N;
  const ModelWeights& m = ctx->ac;
  const auto& D = m.d;
  ctx->clear_taps();
  ctx->tap_enc = w.e.enc; ctx->tap_enc_n = BL * 512;
  ctx->tap_cond = w.cond; ctx->tap_cond_n = BN * 512;
  ctx->tap_melpre = w.melpre; ctx->tap_melpre_n = BN * 80;
  ctx->tap_decout = w.hout; ctx->tap_decout_n = BN * 1024;

  VTTS_CUDA(cudaMemsetAsync(mel, 0, BN * 80 * sizeof(float), st));
  VTTS_CUDA(cudaMemsetAsync(w.melpre, 0, BN * 80 * sizeof(float), st));
  int rc = run_acoustic_front(ctx, tokens, lengths, dur, n_frames, B, L, N, w, st);
  if (rc) return rc;
  // ---- REFERENCE: the 2N prenet sub-keys of the reference's chain, stream-ordered into the workspace ----
  if (mode == VTTS_DROPOUT_REFERENCE) {
    ref_subkey_chain_kernel<<<1, 32, 0, st>>>(seed, 2 * N, w.subkeys);
    ctx->launches++;
    VTTS_CUDA(cudaGetLastError());
  }
  // ---- autoregressive scan: ONE launch for up to DEC_NG * 32 rows (row groups share the grid barriers of a frame) ----
  for (int b0 = 0; b0 < B; b0 += DEC_NG * DEC_XR) {
    const int nb = B - b0 < DEC_NG * DEC_XR ? B - b0 : DEC_NG * DEC_XR;
    DecScanArgs da;
    memset(&da, 0, sizeof(da));
    da.zc0 = w.zc0 + (size_t)b0 * N * 2048; da.zc1 = w.zc1 + (size_t)b0 * N * 2048;
    da.w0r = D[D_DEC_W0R]; da.w1r = D[D_DEC_W1R]; da.wc = D[D_DEC_WC]; da.bc = D[D_DEC_BC]; da.wp2 = D[D_DEC_WP2];
    da.keep = keep; da.subkeys = w.subkeys; da.seed = seed; da.mode = mode;
    da.p1 = w.p1; da.p2 = w.p2; da.h0 = w.h0; da.h1 = w.h1; da.hout = w.hout + (size_t)b0 * N * 1024;
    da.bar = w.dec_bar; da.err = ctx->d_err;
    VTTS_CUDA(cudaMemsetAsync(w.dec_bar, 0, sizeof(unsigned int), st));
    da.B = nb; da.N = N; da.row_base = b0; da.dbg = ctx->tc_dbg_on ? ctx->d_tc_dbg : nullptr;
    void* args[] = {&da};
    VTTS_CUDA(cudaLaunchCooperativeKernel((void*)decoder_scan_kernel<false>, dim3(DEC_CTAS), dim3(SCAN_THREADS), args, dec_scan_smem(), st));
    ctx->launches++;
  }
  ctx->sub_mark(4, st);
  rc = run_projection_postnet(ctx, w.hout, n_frames, B, N, w.melpre, w.q0, w.q1, nullptr, 5, mel, st);
  if (rc) return rc;
  ctx->sub_mark(6, st);
  return VTTS_OK;
}

// the first n sub-keys of the hk.next_rng_key() chain (host side of ref_subkey_chain_kernel, same function)
static void ref_subkeys_host(uint64_t seed, int n, uint2* out) {
  uint32_t k0 = (uint32_t)(seed >> 32), k1 = (uint32_t)seed;
  for (int i = 0; i < n; ++i) {
    uint32_t s0, s1;
    jax_split(k0, k1, s0, s1);
    out[i] = make_uint2(s0, s1);
  }
}

int vtts_teacher_mode_check(vtts_ctx* ctx, int mode, int B, int N) {
  if (mode < VTTS_DROPOUT_OFF || mode > VTTS_DROPOUT_REFERENCE)
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic (teacher forced): dropout_mode %d", mode);
  // the reference's zoneout draws count B*N*512 words with a 32-bit counter
  if (mode == VTTS_DROPOUT_REFERENCE && (uint64_t)B * (uint64_t)N * vc::DEC_H >= (1ull << 32))
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic (teacher forced): REFERENCE draws need B*N*512 < 2^32 (B=%d N=%d)", B, N);
  return VTTS_OK;
}

// AcousticModel.__call__ (model.py:146-169) with is_training=False, as gta.py:24-25 (`val_net`) runs it:
// encoder -> upsample to the mel length -> prenet of the SHIFTED ground-truth mel (dropout live) -> zoneout decoder
// scan -> projection -> postnet.  mel1 = projection output (may be null), mel2 = mel1 + postnet(mel1).
int vtts_acoustic_teacher_run(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur,
                              const int32_t* n_frames, const float* mels_in, const uint8_t* keep, const uint8_t* zone, int mode,
                              uint64_t seed, int B, int L, int N, float* mel1, float* mel2, cudaStream_t st) {
  if (!ctx->ac.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "acoustic weights not loaded");
  if (B < 1 || L < 1 || N < 1 || B > MAX_ROWS)
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic (teacher forced): B=%d L=%d N=%d (1 <= B <= %d rows per call)", B, L, N, MAX_ROWS);
  int rc = vtts_teacher_mode_check(ctx, mode, B, N);
  if (rc) return rc;
  if (mode == VTTS_DROPOUT_MASK && (!keep || !zone))
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic (teacher forced): dropout_mode MASK needs keep_mask and zone_mask");
  if (ctx->sm_count < SCAN_CTAS) return ctx->fail(VTTS_ERR_NO_DEVICE, "scan kernels need %d SMs, device has %d", SCAN_CTAS, ctx->sm_count);
  const TfBufs w = carve_ws<TfBufs>(ctx, B, L, N);
  const size_t BL = (size_t)B * L, BN = (size_t)B * N;
  const ModelWeights& m = ctx->ac;
  const auto& T = m.t;
  const auto& D = m.d;
  ctx->clear_taps();   // cond: the first 512 columns of dec_in
  ctx->tap_enc = w.e.enc; ctx->tap_enc_n = BL * 512;
  ctx->tap_melpre = w.melpre; ctx->tap_melpre_n = BN * 80;
  ctx->tap_decin = w.xin; ctx->tap_decin_n = BN * XW;
  ctx->tap_decout = w.hout; ctx->tap_decout_n = BN * 1024;
  VTTS_CUDA(cudaMemsetAsync(mel2, 0, BN * 80 * sizeof(float), st));
  if (mel1) VTTS_CUDA(cudaMemsetAsync(mel1, 0, BN * 80 * sizeof(float), st));
  VTTS_CUDA(cudaMemsetAsync(w.xin, 0, BN * XW * sizeof(float), st));
  VTTS_CUDA(cudaMemsetAsync(w.melpre, 0, BN * 80 * sizeof(float), st));
  // REFERENCE: the six sub-keys of AcousticModel.__call__ (two prenet dropouts, then the zoneout draws h0, c0, h1, c1)
  uint2 rk[6] = {};
  if (mode == VTTS_DROPOUT_REFERENCE) ref_subkeys_host(seed, 6, rk);
  ctx->sub_mark(16, st);
  rc = run_token_encoder(ctx, m, tokens, lengths, B, L, w.e, st);
  if (rc) return rc;
  rc = run_upsample(ctx, w.e.enc, dur, lengths, n_frames, B, L, N, w.xin, XW, st);   // cond -> columns 0..511 of the decoder input
  if (rc) return rc;
  ctx->sub_mark(17, st);
  // ---- prenet over the whole sequence (model.py:95-100,149): two bias-free linears, relu, dropout 0.5 each ----
  const size_t act_blocks = (BN * 256 + 255) / 256;
  const unsigned act_grid = (unsigned)(act_blocks < ctx->sm_count * 16 ? act_blocks : ctx->sm_count * 16);
  const ConvProb pre1 = conv_prob(mels_in, T[aci::PRE1_W], D[D_ZERO], w.pa);
  rc = run_convs(ctx, &pre1, 1, 80, 256, 1, (int)BN, nullptr, 0, m.tiles(PK_PRE1), st);
  if (rc) return rc;
  prenet_act_kernel<<<act_grid, 256, 0, st>>>(w.pa, keep, seed, mode, rk[0], 0, B, N, w.pb, 256);
  ctx->launches++;
  const ConvProb pre2 = conv_prob(w.pb, T[aci::PRE2_W], D[D_ZERO], w.pa);
  rc = run_convs(ctx, &pre2, 1, 256, 256, 1, (int)BN, nullptr, 0, m.tiles(PK_PRE2), st);
  if (rc) return rc;
  prenet_act_kernel<<<act_grid, 256, 0, st>>>(w.pa, keep, seed, mode, rk[1], 1, B, N, w.xin + vc::ENC_OUT, XW);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  // ---- every input-side product of both LSTMs in one launch: zc = [cond | p2] . W[0:768] + b ----
  const ConvProb hp[2] = {conv_prob(w.xin, T[aci::DEC_L0_W], T[aci::DEC_L0_B], w.zc0), conv_prob(w.xin, T[aci::DEC_L1_W], T[aci::DEC_L1_B], w.zc1)};
  rc = run_convs(ctx, hp, 2, XW, 2048, 1, (int)BN, nullptr, 0, m.tiles(PK_TF_L0), st);
  if (rc) return rc;
  ctx->sub_mark(18, st);
  // ---- zoneout scan, <= 32 rows per launch ----
  for (int b0 = 0; b0 < B; b0 += DEC_XR) {
    const int nb = B - b0 < DEC_XR ? B - b0 : DEC_XR;
    TfScanArgs ta;
    memset(&ta, 0, sizeof(ta));
    ta.zc0 = w.zc0 + (size_t)b0 * N * 2048; ta.zc1 = w.zc1 + (size_t)b0 * N * 2048;
    ta.w0r = D[D_DEC_W0R]; ta.w1r = D[D_DEC_W1R];
    ta.zone = zone; ta.seed = seed; ta.mode = mode;
    for (int i = 0; i < 4; ++i) ta.zkey[i] = rk[2 + i];
    ta.h0s = w.h0s; ta.h1s = w.h1s; ta.hout = w.hout + (size_t)b0 * N * 1024;
    ta.B = nb; ta.N = N; ta.row_base = b0; ta.B_call = B;
    void* args[] = {&ta};
    VTTS_CUDA(cudaLaunchCooperativeKernel((void*)decoder_tf_scan_kernel, dim3(SCAN_CTAS), dim3(SCAN_THREADS), args, tf_scan_smem(), st));
    ctx->launches++;
  }
  ctx->sub_mark(19, st);
  rc = run_projection_postnet(ctx, w.hout, n_frames, B, N, w.melpre, w.q0, w.q1, mel1, -1, mel2, st);
  ctx->sub_mark(20, st);
  return rc;
}

// Test hook: the masks REFERENCE mode applies, drawn on the device by the functions the scans call.
int vtts_debug_dropout_masks(vtts_ctx* ctx, int kind, uint64_t seed, int B, int N, uint8_t* host_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!host_out || (kind != 0 && kind != 1) || N < 1 || (kind == 1 && B < 1))
    return ctx->fail(VTTS_ERR_BAD_ARG, "debug_dropout_masks: kind=%d B=%d N=%d", kind, B, N);
  if (kind == 1) {
    const int rc = vtts_teacher_mode_check(ctx, VTTS_DROPOUT_REFERENCE, B, N);
    if (rc) return rc;
  }
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t nk = (size_t)(kind == 0 ? 1 : B) * N * 2 * vc::PRENET, nz = kind == 0 ? 0 : (size_t)B * N * 4 * vc::DEC_H;
  Arena sz(nullptr, 0, true);
  sz.take<uint2>((size_t)2 * N);
  sz.take<uint8_t>(nk + nz);
  int rc = ctx->ensure_ws(sz.off + 256);
  if (rc) return rc;
  Arena ar(ctx->ws, ctx->ws_bytes, false);
  uint2* subkeys = ar.take<uint2>((size_t)2 * N);
  uint8_t* d = ar.take<uint8_t>(nk + nz);
  const size_t blocks = (nk + nz + 255) / 256;
  const unsigned grid = (unsigned)(blocks < (size_t)ctx->sm_count * 16 ? blocks : (size_t)ctx->sm_count * 16);
  if (kind == 0) {
    ref_subkey_chain_kernel<<<1, 32>>>(seed, 2 * N, subkeys);
    ref_ar_masks_kernel<<<grid, 256>>>(subkeys, N, d);
  } else {
    uint2 rk[6];
    ref_subkeys_host(seed, 6, rk);
    ref_tf_masks_kernel<<<grid, 256>>>(rk[0], rk[1], rk[2], rk[3], rk[4], rk[5], B, N, d, d + nk);
  }
  VTTS_CUDA(cudaGetLastError());
  VTTS_CUDA(cudaDeviceSynchronize());
  VTTS_CUDA(cudaMemcpy(host_out, d, nk + nz, cudaMemcpyDeviceToHost));
  return VTTS_OK;
}

// =====================================================================================================
// DurationModel (vietTTS/nat/model.py:49-70): TokenEncoder -> Linear(512->256) -> gelu -> Linear(256->1) -> softplus.
// The encoder is run_token_encoder above with the duration checkpoint's weights; the first Linear is a k=1
// contraction through the shared conv dispatch; the head below finishes gelu / dot / softplus per token.
// =====================================================================================================
namespace {

// jax.nn.gelu default (approximate=True): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
__device__ __forceinline__ float gelu_tanh(float x) {
  const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  return 0.5f * x * (1.f + tanhf(u));
}
// jax.nn.softplus = logaddexp(x, 0)
__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// one warp per token: y [BL][256] (pre-activation of the first Linear, bias included) -> dur[BL] seconds
__global__ void __launch_bounds__(256) duration_head_kernel(const float* __restrict__ y, const float* __restrict__ w2,
                                                            const float* __restrict__ b2, const int32_t* __restrict__ lengths,
                                                            int B, int L, float* __restrict__ dur) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tok = blockIdx.x * 8 + warp;
  if (tok >= B * L) return;
  const int b = tok / L, l = tok - b * L;
  if (lengths && l >= lengths[b]) {
    if (lane == 0) dur[tok] = 0.f;
    return;
  }
  const float* yr = y + (size_t)tok * 256 + lane * 8;
  const float4 a0 = __ldg(reinterpret_cast<const float4*>(yr)), a1 = __ldg(reinterpret_cast<const float4*>(yr + 4));
  const float4 w0 = __ldg(reinterpret_cast<const float4*>(w2 + lane * 8)), w1 = __ldg(reinterpret_cast<const float4*>(w2 + lane * 8 + 4));
  float s = gelu_tanh(a0.x) * w0.x;
  s = fmaf(gelu_tanh(a0.y), w0.y, s);
  s = fmaf(gelu_tanh(a0.z), w0.z, s);
  s = fmaf(gelu_tanh(a0.w), w0.w, s);
  s = fmaf(gelu_tanh(a1.x), w1.x, s);
  s = fmaf(gelu_tanh(a1.y), w1.y, s);
  s = fmaf(gelu_tanh(a1.z), w1.z, s);
  s = fmaf(gelu_tanh(a1.w), w1.w, s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) dur[tok] = softplus(s + __ldg(b2));
}

// packing table of the duration model (ctx->du.tiles)
enum { PK_DU_FC1 = PK_ENC_COUNT, PK_DU_COUNT };

}  // namespace

int vtts_duration_prepare(vtts_ctx* ctx) {
  ModelWeights& m = ctx->du;
  std::vector<size_t> dn(D_ENC_COUNT);
  std::vector<PackSpec> pk(PK_DU_COUNT);
  encoder_tables(m, dn, pk);
  pk[PK_DU_FC1] = {m.t[dui::FC1_W], 1, 512, 256};
  int rc = vtts_alloc_tensors(ctx, dn, &m.derived, m.d);
  if (rc) return rc;
  encoder_derive(m);
  VTTS_CUDA(cudaGetLastError());
  rc = vtts_pack_convs(ctx, m, pk);
  if (rc) return rc;
  VTTS_CUDA(cudaDeviceSynchronize());
  VTTS_CUDA(cudaFuncSetAttribute(enc_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)enc_scan_smem()));
  return VTTS_OK;
}

int vtts_duration_run(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float* dur_sec,
                      cudaStream_t st) {
  if (!ctx->du.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "duration weights not loaded");
  if (B < 1 || L < 1 || B > MAX_ROWS)
    return ctx->fail(VTTS_ERR_BAD_ARG, "duration: B=%d L=%d (1 <= B <= %d rows per call; the host layer chunks larger batches)", B, L, MAX_ROWS);
  if (ctx->sm_count < SCAN_CTAS) return ctx->fail(VTTS_ERR_NO_DEVICE, "scan kernels need %d SMs, device has %d", SCAN_CTAS, ctx->sm_count);
  const DuBufs w = carve_ws<DuBufs>(ctx, B, L, 0);
  const size_t BL = (size_t)B * L;
  const ModelWeights& m = ctx->du;
  ctx->clear_taps();
  ctx->tap_enc = w.e.enc; ctx->tap_enc_n = BL * 512;
  ctx->tap_durhid = w.y; ctx->tap_durhid_n = BL * 256;
  // padded encoder rows are never written by the scan: clear them so the projection reads zeros, not stale workspace
  VTTS_CUDA(cudaMemsetAsync(w.e.enc, 0, BL * 512 * sizeof(float), st));
  int rc = run_token_encoder(ctx, m, tokens, lengths, B, L, w.e, st);
  if (rc) return rc;
  // ---- projection head ----
  const ConvProb p = conv_prob(w.e.enc, m.t[dui::FC1_W], m.t[dui::FC1_B], w.y);
  rc = run_convs(ctx, &p, 1, 512, 256, 1, (int)BL, nullptr, 0, m.tiles(PK_DU_FC1), st);
  if (rc) return rc;
  duration_head_kernel<<<(unsigned)((BL + 7) / 8), 256, 0, st>>>(w.y, m.t[dui::FC2_W], m.t[dui::FC2_B], lengths, B, L, dur_sec);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}
