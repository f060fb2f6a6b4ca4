// HiFiGAN generator forward -- restates Generator.__call__ (vietTTS/hifigan/model.py:109-125) on top of the generic
// conv kernel (strict fp32) or the tensor-core kernels of tc_conv.cu (bf16x3, or fp16 in VTTS_PRECISION_FP16).
//
//   conv_pre                              model.py:110
//   per stage: lrelu(0.1) -> ups[i]       model.py:112-114   (u output phases, 2 taps each; one dense conv over blocks of
//                                                               u output rows on the tensor cores)
//              3 x ResBlock1, mean        model.py:115-121   (mean fused into the next consumer)
//   lrelu(0.01) -> conv_post -> tanh      model.py:122-124   (conv_post_kernel below)
#include "vtts_internal.cuh"

using namespace hgpk;

namespace {

// ---- ConvTranspose weight repack: Haiku w[K][Cout][Cin] -> per phase r: [2][Cin][Cout] ----------
// hk.Conv1DTranspose("SAME"): y[t,o] = b[o] + sum_j sum_i xdpad[t+j, i] w[j,o,i] with the input
// zero-dilated by `u` and padded by a = ceil((K+u-2)/2) on the left.  For t = tau*u + r only taps
// j = j0 + q*u (q = 0,1; j0 = (a - r) mod u) hit a non-zero sample, x[tau + e + q], e = (r + j0 - a)/u.
__global__ void repack_ups_kernel(const float* __restrict__ w, float* __restrict__ out, int u, int K, int Cin, int Cout, int a) {
  const size_t total = (size_t)u * 2 * Cin * Cout;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int o = idx % Cout;
    int i = (idx / Cout) % Cin;
    int q = (idx / ((size_t)Cout * Cin)) % 2;
    int r = idx / ((size_t)Cout * Cin * 2);
    int j0 = ((a - r) % u + u) % u;
    int j = j0 + q * u;
    out[idx] = w[((size_t)j * Cout + o) * Cin + i];
  }
}

// conv_post: out[b,t] = tanh(bias + sum_{j<7} sum_{i<32} lrelu_0.01(mean3(x)[t+j-3, i]) w[j,i])
__global__ void __launch_bounds__(256) conv_post_kernel(const float* __restrict__ a0, const float* __restrict__ a1,
                                                        const float* __restrict__ a2, const float* __restrict__ w,
                                                        const float* __restrict__ bias, const int* __restrict__ len,
                                                        int len_mul, int R, float* __restrict__ wav) {
  constexpr int C = 32, KW = 7, TT = 256, ST = 33;
  __shared__ float xs[(TT + KW - 1) * ST];
  __shared__ float wsm[KW * C];
  const int b = blockIdx.y, t0 = blockIdx.x * TT, tid = threadIdx.x;
  int valid = R;
  if (len) {
    int v = len[b] * len_mul;
    valid = v < valid ? v : valid;
  }
  if (tid < KW * C) wsm[tid] = w[tid];
  const size_t base = (size_t)b * R * C;
  if (t0 < valid) {
    for (int e = tid; e < (TT + KW - 1) * (C / 4); e += 256) {
      int rr = e / (C / 4), q = e % (C / 4);
      int r = t0 - 3 + rr;
      float4 v = make_float4(0, 0, 0, 0);
      if (r >= 0 && r < valid) {
        size_t off = base + (size_t)r * C + q * 4;
        float4 x = __ldg(reinterpret_cast<const float4*>(a0 + off));
        float4 y = __ldg(reinterpret_cast<const float4*>(a1 + off));
        float4 z = __ldg(reinterpret_cast<const float4*>(a2 + off));
        v.x = ((x.x + y.x) + z.x) / 3.0f;
        v.y = ((x.y + y.y) + z.y) / 3.0f;
        v.z = ((x.z + y.z) + z.z) / 3.0f;
        v.w = ((x.w + y.w) + z.w) / 3.0f;
        v.x = v.x >= 0.f ? v.x : 0.01f * v.x;
        v.y = v.y >= 0.f ? v.y : 0.01f * v.y;
        v.z = v.z >= 0.f ? v.z : 0.01f * v.z;
        v.w = v.w >= 0.f ? v.w : 0.01f * v.w;
      }
      float* d = xs + rr * ST + q * 4;
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
  }
  __syncthreads();
  const int t = t0 + tid;
  if (t >= R) return;
  float out = 0.f;
  if (t < valid) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < KW; ++j)
#pragma unroll
      for (int i = 0; i < C; ++i) acc = fmaf(xs[(tid + j) * ST + i], wsm[j * C + i], acc);
    out = tanhf(acc + bias[0]);
  }
  wav[(size_t)b * R + t] = out;
}

struct HgBufs {
  float* P0;        // conv_pre out [B][T][512]
  float* A[2][3];   // resblock outputs (alternate by stage parity)
  float* X;         // ups out
  float* Tb[3];     // conv1 out
  float* Bb[3];     // ping-pong
};

void carve(Arena& ar, int B, int T, HgBufs& hb) {
  const size_t frames = (size_t)B * T;
  hb.P0 = ar.take<float>(frames * 512);
  const size_t big = frames * 8192;
  for (int p = 0; p < 2; ++p)
    for (int j = 0; j < 3; ++j) hb.A[p][j] = ar.take<float>(big);
  hb.X = ar.take<float>(big);
  for (int j = 0; j < 3; ++j) hb.Tb[j] = ar.take<float>(big);
  for (int j = 0; j < 3; ++j) hb.Bb[j] = ar.take<float>(big);
}

}  // namespace

size_t vtts_hifigan_ws_bytes(int B, int T) {
  Arena ar(nullptr, 0, true);
  HgBufs hb;
  carve(ar, B, T, hb);
  return ar.off + 256;
}

int vtts_hifigan_prepare(vtts_ctx* ctx) {
  ModelWeights& m = ctx->hg;
  // derived, per stage i: the transposed-conv weights repacked per output phase, [u][2][C][C/2] (D_UPS_PH, the strict
  // fp32 path), the same stacked per block of u output rows, [2][C][u][C/2] (D_UPS_BLK, see hg_ups), and the bias
  // repeated per output row of the block, [u][C/2] (D_UPS_BLK_B)
  std::vector<size_t> dn(12);
  for (int i = 0, C = vc::HG_C0; i < 4; ++i, C /= 2) {
    dn[D_UPS_PH(i)] = dn[D_UPS_BLK(i)] = (size_t)vc::hg_rate(i) * 2 * C * (C / 2);
    dn[D_UPS_BLK_B(i)] = (size_t)vc::hg_rate(i) * (C / 2);
  }
  int rc = vtts_alloc_tensors(ctx, dn, &m.derived, m.d);
  if (rc) return rc;
  std::vector<PackSpec> pk(2 * PK_COUNT);
  for (int i = 0, C = vc::HG_C0; i < 4; ++i, C /= 2) {
    const int u = vc::hg_rate(i), K = vc::hg_upk(i), Co = C / 2;
    repack_ups_kernel<<<256, 256>>>(m.t[hgi::UPS_W(i)], m.d[D_UPS_PH(i)], u, K, C, Co, (K + u - 2 + 1) / 2);
    VTTS_CUDA(cudaGetLastError());
    // column block mm of the block weights is phase (mm + u/2) mod u: the first half of a block holds the late phases
    // of one input row, the second half the early phases of the next
    for (int mm = 0; mm < u; ++mm) {
      const int r = (mm + u / 2) % u;
      VTTS_CUDA(cudaMemcpy2D(m.d[D_UPS_BLK(i)] + (size_t)mm * Co, (size_t)u * Co * 4, m.d[D_UPS_PH(i)] + (size_t)r * 2 * C * Co, (size_t)Co * 4,
                             (size_t)Co * 4, 2 * C, cudaMemcpyDeviceToDevice));
      VTTS_CUDA(cudaMemcpy(m.d[D_UPS_BLK_B(i)] + (size_t)mm * Co, m.t[hgi::UPS_B(i)], (size_t)Co * 4, cudaMemcpyDeviceToDevice));
    }
    pk[PK_UPS(i)] = {m.d[D_UPS_BLK(i)], 2, C, u * Co};
  }
  for (int n = 0; n < 12; ++n)
    for (int which = 0; which < 2; ++which)
      for (int j = 0; j < 3; ++j) {
        const int ch = 256 >> (n / 3);
        pk[PK_RB(n, which, j)] = {m.t[hgi::RB_W(n, which, j)], vc::hg_rbk(n % 3), ch, ch};
      }
  pk[PK_PRE] = {m.t[hgi::PRE_W], 7, vc::MEL, vc::HG_C0};
  for (int e = 0; e < PK_COUNT; ++e) {
    pk[PK_COUNT + e] = pk[e];
    pk[PK_COUNT + e].f16 = true;
  }
  // ---- tensor-core path: bf16 hi/lo split (and fp16) + canonical K-major packing of every dense conv ----
  VTTS_CUDA(cudaDeviceSynchronize());  // the block weights are packed from the repacked transposed-conv weights
  rc = vtts_pack_convs(ctx, m, pk);
  if (rc) return rc;
  VTTS_CUDA(cudaDeviceSynchronize());
  return VTTS_OK;
}

// ---- the generator's layers, one function each: vtts_hifigan_run calls them in order, vtts_debug_hifigan_layer one ----
// Every layer derives its rows from T mel frames and its valid rows from n_frames[b]: stage i runs on T * hg_scale(i)
// input rows per batch row, and rows at or past n_frames[b] * hg_scale(i) read as zero and are not written.

namespace {

// rows per mel frame entering stage i (i = 4: conv_post)
int hg_scale(int i) {
  int s = 1;
  for (int q = 0; q < i; ++q) s *= vc::hg_rate(q);
  return s;
}

// conv_pre: 80 -> 512, k7 pad 3.  mel [B][T][80] -> out [B][T][512]
int hg_conv_pre(vtts_ctx* ctx, const float* mel, float* out, const int32_t* n_frames, int B, int T, cudaStream_t st) {
  const ModelWeights& M = ctx->hg;
  auto& W = M.t;
  ConvLaunch L;
  memset(&L, 0, sizeof(L));
  L.B = B;
  L.len = n_frames;
  L.nprob = 1;
  L.Cin = vc::MEL; L.Cout = vc::HG_C0;
  L.T_rows = T; L.rows_out = T; L.len_mul = 1;
  L.pre_mode = 0; L.pre_slope = 1.f; L.post_act = 0;
  L.p[0] = ConvProb{mel, nullptr, nullptr, W[hgi::PRE_W], W[hgi::PRE_B], nullptr, nullptr, nullptr, nullptr, out, 7, 1, -3, 1, 0};
  // tensor-core modes: bf16x3 (BF16X3) or one fp16 product (FP16, the packing table's second half)
  const bool tc = ctx->precision != VTTS_PRECISION_FP32;
  const int f16 = ctx->precision == VTTS_PRECISION_FP16;
  const int pk = f16 ? PK_COUNT : 0;
  if (!tc) return vtts_launch_conv(ctx, L, st);
  TcLaunch TL;
  memset(&TL, 0, sizeof(TL));
  TL.nprob = 2; TL.Cin = vc::MEL; TL.N = 256; TL.in_ld = vc::MEL; TL.out_ld = vc::HG_C0;
  TL.B = B; TL.T_rows = T; TL.rows_out = T; TL.len = n_frames; TL.len_mul = 1; TL.pre_mode = 0; TL.pre_slope = 1.f; TL.f16 = f16;
  for (int t = 0; t < 2; ++t)
    TL.p[t] = TcProb{mel, nullptr, nullptr, M.tiles(pk + PK_PRE)[t], W[hgi::PRE_B] + 256 * t, nullptr, nullptr, nullptr, nullptr, out + 256 * t, 7, 1, -3, 1, 0};
  return vtts_launch_tc_conv(ctx, TL, st);
}

// lrelu(0.1) [of the 3-way mean for i > 0] -> ConvTranspose of stage i as u two-tap phases.  x[0] (i = 0: conv_pre's
// output) or x[0..2] (the previous stage's three ResBlock chains), [B][T*hg_scale(i)][C] -> out [B][T*hg_scale(i+1)][C/2]
int hg_ups(vtts_ctx* ctx, int i, const float* const* x, float* out, const int32_t* n_frames, int B, int T, cudaStream_t st) {
  const ModelWeights& M = ctx->hg;
  auto& W = M.t;
  const bool tc = ctx->precision != VTTS_PRECISION_FP32;
  const int f16 = ctx->precision == VTTS_PRECISION_FP16;
  const int pk = f16 ? PK_COUNT : 0;
  const int C = vc::HG_C0 >> i, scale_in = hg_scale(i), rows_in = T * scale_in;
  const int u = vc::hg_rate(i), K = vc::hg_upk(i), Co = C / 2;
  const int a = (K + u - 2 + 1) / 2;
  ConvLaunch L;
  memset(&L, 0, sizeof(L));
  L.B = B; L.len = n_frames; L.len_mul = scale_in;
  L.nprob = u; L.Cin = C; L.Cout = Co;
  L.T_rows = rows_in; L.rows_out = rows_in * u;
  L.pre_mode = (i == 0) ? 1 : 2; L.pre_slope = 0.1f; L.post_act = 0;
  for (int r = 0; r < u; ++r) {
    int j0 = ((a - r) % u + u) % u;
    int e = (r + j0 - a) / u;  // exact division, <= 0
    ConvProb p;
    memset(&p, 0, sizeof(p));
    if (i == 0) { p.x0 = x[0]; } else { p.x0 = x[0]; p.x1 = x[1]; p.x2 = x[2]; }
    p.w = M.d[D_UPS_PH(i)] + (size_t)r * 2 * C * Co;
    p.bias = W[hgi::UPS_B(i)];
    p.out = out;
    p.k = 2; p.dil = 1; p.in_off = e; p.out_stride = u; p.out_off = r;
    L.p[r] = p;
  }
  if (!tc) return vtts_launch_conv(ctx, L, st);
  // Tensor cores: one dense two-tap conv over blocks of u output rows, so that every output phase shares one converted
  // activation tile.  Phase r of input row tau reads x[tau - 1 + q] for r < u/2 and x[tau + q] for r >= u/2 (q = 0, 1),
  // so block s, output rows u*s - u/2 .. u*s + u/2 - 1 (phases u/2.. of row s - 1, then phases ..u/2 - 1 of row s),
  // reads x[s - 1] and x[s] with the stacked weights D_UPS_BLK: in_off = -1 over s = 0..rows_in.  In the [B][u*rows_in]
  // [Co] output a block is one row of u*Co floats starting u/2 output rows early (out_e0); N <= 256 columns per problem.
  const int N = vtts_tc_tile_n(u * Co), nt = u * Co / N;
  TcLaunch TL;
  memset(&TL, 0, sizeof(TL));
  TL.nprob = nt; TL.Cin = C; TL.N = N; TL.in_ld = C; TL.out_ld = u * Co; TL.out_sub = Co;
  TL.B = B; TL.T_rows = rows_in; TL.rows_out = rows_in * u; TL.tile_rows = rows_in + 1; TL.len = n_frames; TL.len_mul = scale_in;
  TL.pre_mode = L.pre_mode; TL.pre_slope = 0.1f; TL.f16 = f16;
  for (int g = 0; g < nt; ++g) {
    TcProb& q = TL.p[g];
    q.x0 = L.p[0].x0; q.x1 = L.p[0].x1; q.x2 = L.p[0].x2;
    q.wpk = M.tiles(pk + PK_UPS(i))[g]; q.bias = M.d[D_UPS_BLK_B(i)] + g * N; q.out = out;
    q.k = 2; q.dil = 1; q.in_off = -1; q.out_stride = 1; q.out_off = 0; q.out_e0 = -(u / 2) * Co + g * N;
  }
  return vtts_launch_tc_conv(ctx, TL, st);
}

// step m of the three ResBlock1 (k = 3, 7, 11) of stage i: chain j runs dst[j] = conv2(lrelu(conv1_d(lrelu(src[j])))) +
// src[j], all [B][T*hg_scale(i+1)][C/2]; tmp[j] receives conv1's output when the pair is not fused
int hg_resblock(vtts_ctx* ctx, int i, int m, const float* const* src, float* const* dst, float* const* tmp, const int32_t* n_frames,
                int B, int T, cudaStream_t st) {
  const ModelWeights& M = ctx->hg;
  auto& W = M.t;
  const bool tc = ctx->precision != VTTS_PRECISION_FP32;
  const int f16 = ctx->precision == VTTS_PRECISION_FP16;
  const int pk = f16 ? PK_COUNT : 0;
  const int Co = vc::HG_C0 >> (i + 1), scale = hg_scale(i + 1), rows = T * scale;
  const int d = vc::hg_dil(m);
  if (tc && ctx->fuse_pairs && Co <= 64) {
    // ---- fused pair: conv(d) -> lrelu -> conv(1) -> + x, intermediate kept on chip (tc_conv.cu) ----
    TcPairLaunch PL;
    memset(&PL, 0, sizeof(PL));
    PL.nprob = 3; PL.N = Co; PL.B = B; PL.T_rows = rows; PL.len = n_frames; PL.len_mul = scale; PL.slope = 0.1f; PL.f16 = f16;
    for (int j = 0; j < 3; ++j) {
      const int kk = vc::hg_rbk(j), n = i * 3 + j;
      PL.p[j] = TcPairProb{src[j], M.tiles(pk + PK_RB(n, 0, m))[0], M.tiles(pk + PK_RB(n, 1, m))[0], W[hgi::RB_B(n, 0, m)], W[hgi::RB_B(n, 1, m)],
                           dst[j], kk, d};
    }
    return vtts_launch_tc_pair(ctx, PL, st);
  }
  if (tc) {
    // ---- tensor-core path (tc_conv.cu) ----
    TcLaunch TL;
    for (int which = 0; which < 2; ++which) {
      memset(&TL, 0, sizeof(TL));
      TL.nprob = 3; TL.Cin = Co; TL.N = Co; TL.in_ld = Co; TL.out_ld = Co;
      TL.B = B; TL.T_rows = rows; TL.rows_out = rows; TL.len = n_frames; TL.len_mul = scale;
      TL.pre_mode = 1; TL.pre_slope = 0.1f; TL.f16 = f16;
      for (int j = 0; j < 3; ++j) {
        const int kk = vc::hg_rbk(j), n = i * 3 + j;
        const int dd = which == 0 ? d : 1;
        TcProb p;
        memset(&p, 0, sizeof(p));
        p.x0 = which == 0 ? src[j] : tmp[j];
        p.wpk = M.tiles(pk + PK_RB(n, which, m))[0];
        p.bias = W[hgi::RB_B(n, which, m)];
        p.resid = which == 0 ? nullptr : src[j];
        p.out = which == 0 ? tmp[j] : dst[j];
        p.k = kk; p.dil = dd; p.in_off = -((kk - 1) * dd) / 2; p.out_stride = 1; p.out_off = 0;
        TL.p[j] = p;
      }
      int rc = vtts_launch_tc_conv(ctx, TL, st);
      if (rc) return rc;
    }
    return VTTS_OK;
  }
  // conv1 (dilated)
  ConvLaunch L;
  memset(&L, 0, sizeof(L));
  L.B = B; L.len = n_frames; L.len_mul = scale;
  L.nprob = 3; L.Cin = Co; L.Cout = Co; L.T_rows = rows; L.rows_out = rows;
  L.pre_mode = 1; L.pre_slope = 0.1f; L.post_act = 0;
  for (int j = 0; j < 3; ++j) {
    const int kk = vc::hg_rbk(j), n = i * 3 + j;
    ConvProb p;
    memset(&p, 0, sizeof(p));
    p.x0 = src[j];
    p.w = W[hgi::RB_W(n, 0, m)]; p.bias = W[hgi::RB_B(n, 0, m)];
    p.out = tmp[j];
    p.k = kk; p.dil = d; p.in_off = -((kk - 1) * d) / 2; p.out_stride = 1; p.out_off = 0;
    L.p[j] = p;
  }
  int rc = vtts_launch_conv(ctx, L, st);
  if (rc) return rc;
  // conv2 (dilation 1) + residual
  for (int j = 0; j < 3; ++j) {
    const int kk = vc::hg_rbk(j), n = i * 3 + j;
    ConvProb p;
    memset(&p, 0, sizeof(p));
    p.x0 = tmp[j];
    p.w = W[hgi::RB_W(n, 1, m)]; p.bias = W[hgi::RB_B(n, 1, m)];
    p.resid = src[j];
    p.out = dst[j];
    p.k = kk; p.dil = 1; p.in_off = -(kk - 1) / 2; p.out_stride = 1; p.out_off = 0;
    L.p[j] = p;
  }
  return vtts_launch_conv(ctx, L, st);
}

// mean of 3, lrelu(0.01), conv_post (32 -> 1, k7), tanh: x[0..2] [B][256T][32] -> wav [B][256T], zeros past
// n_frames[b] * 256
int hg_conv_post(vtts_ctx* ctx, const float* const* x, float* wav, const int32_t* n_frames, int B, int T, cudaStream_t st) {
  auto& W = ctx->hg.t;
  const int R = T * hg_scale(4);  // 256*T
  dim3 grid((R + 255) / 256, B);
  conv_post_kernel<<<grid, 256, 0, st>>>(x[0], x[1], x[2], W[hgi::POST_W], W[hgi::POST_B], n_frames, 256, R, wav);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

int hg_check(vtts_ctx* ctx, int B, int T) {
  if (!ctx->hg.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "hifigan weights not loaded");
  if (B < 1 || T < 1 || B > 65535) return ctx->fail(VTTS_ERR_BAD_ARG, "hifigan: B=%d T=%d", B, T);
  if ((int64_t)T * 256 > (int64_t)INT32_MAX / 64) return ctx->fail(VTTS_ERR_BAD_ARG, "hifigan: T=%d too long", T);
  return VTTS_OK;
}

}  // namespace

int vtts_hifigan_run(vtts_ctx* ctx, const float* mel, const int32_t* n_frames, int B, int T, float* wav, cudaStream_t st) {
  int rc = hg_check(ctx, B, T);
  if (rc) return rc;
  size_t need = vtts_hifigan_ws_bytes(B, T);
  rc = ctx->ensure_ws(need);
  if (rc) return rc;
  Arena ar(ctx->ws, ctx->ws_bytes, false);
  HgBufs hb;
  carve(ar, B, T, hb);

  ctx->sub_mark(8, st);
  rc = hg_conv_pre(ctx, mel, hb.P0, n_frames, B, T, st);
  if (rc) return rc;
  ctx->sub_mark(9, st);
  for (int i = 0; i < 4; ++i) {
    const int par = i & 1;   // stage i's ResBlock chains end in A[par]; stage i - 1's in A[par ^ 1]
    const float* const ups_in[3] = {i == 0 ? hb.P0 : hb.A[par ^ 1][0], i == 0 ? nullptr : hb.A[par ^ 1][1], i == 0 ? nullptr : hb.A[par ^ 1][2]};
    rc = hg_ups(ctx, i, ups_in, hb.X, n_frames, B, T, st);
    if (rc) return rc;
    for (int m = 0; m < 3; ++m) {
      const float* src[3];
      float* dst[3];
      for (int j = 0; j < 3; ++j) {
        src[j] = (m == 0) ? hb.X : (m == 1 ? hb.A[par][j] : hb.Bb[j]);
        dst[j] = (m == 1) ? hb.Bb[j] : hb.A[par][j];
      }
      rc = hg_resblock(ctx, i, m, src, dst, hb.Tb, n_frames, B, T, st);
      if (rc) return rc;
    }
    ctx->sub_mark(10 + i, st);
  }
  rc = hg_conv_post(ctx, hb.A[1], wav, n_frames, B, T, st);
  if (rc) return rc;
  ctx->sub_mark(14, st);
  return VTTS_OK;
}

int vtts_debug_hifigan_layer(vtts_ctx* ctx, int layer, const float* const* x, float* const* out, const int32_t* n_frames, int B, int T) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = hg_check(ctx, B, T);
  if (rc) return rc;
  if (layer < 0 || layer > 17 || !x || !out) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_hifigan_layer: layer %d (0..17), x and out required", layer);
  const int nx = layer <= 1 ? 1 : 3, nout = (layer >= 5 && layer <= 16) ? 3 : 1;
  for (int j = 0; j < nx; ++j)
    if (!x[j]) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_hifigan_layer: layer %d needs %d inputs", layer, nx);
  for (int j = 0; j < nout; ++j)
    if (!out[j]) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_hifigan_layer: layer %d needs %d outputs", layer, nout);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, nullptr);
  if (layer == 0) {
    rc = hg_conv_pre(ctx, x[0], out[0], n_frames, B, T, nullptr);
  } else if (layer <= 4) {
    rc = hg_ups(ctx, layer - 1, x, out[0], n_frames, B, T, nullptr);
  } else if (layer <= 16) {
    // conv1's outputs of the unfused pair: three buffers of the step's shape
    const int i = (layer - 5) / 3, m = (layer - 5) % 3;
    const size_t n = (size_t)B * T * hg_scale(i + 1) * (vc::HG_C0 >> (i + 1));
    float* tmp = nullptr;
    VTTS_CUDA(cudaMalloc(&tmp, 3 * n * sizeof(float)));
    float* const t3[3] = {tmp, tmp + n, tmp + 2 * n};
    rc = hg_resblock(ctx, i, m, x, out, t3, n_frames, B, T, nullptr);
    const cudaError_t e = cudaDeviceSynchronize();
    cudaFree(tmp);
    if (!rc && e != cudaSuccess) return ctx->fail(VTTS_ERR_CUDA, "debug_hifigan_layer: %s", cudaGetErrorString(e));
  } else {
    rc = hg_conv_post(ctx, x, out[0], n_frames, B, T, nullptr);
  }
  if (rc) return rc;
  VTTS_CUDA(cudaDeviceSynchronize());
  return VTTS_OK;
}
