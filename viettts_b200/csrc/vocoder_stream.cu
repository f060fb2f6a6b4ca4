// Stateful streaming generator: mel frames are pushed per stream slot as they arrive, every layer keeps the context it
// needs between pushes, and each push returns the waveform frames whose receptive field is complete.  The layers are
// those of vtts_hifigan_run (tensor-core path, C <= 64 ResBlock pairs as two tc_conv launches each); the emitted samples
// are bit-identical to the one-shot generator with fused pairs off.
//
// Windows.  Every tensor of the generator (mel, conv_pre out, per stage the ConvTranspose out X and, per ResBlock chain j
// and pair m, the conv1 out T and the pair out Y) has one window per slot, [cap][C] floats with cap = lead + rate * F.
// All tensors of one rate share the map  time t  <->  window row  t - rate * P_old + lead(rate),  P_old = frames the slot
// received before this push.  A tensor with lag g (its rows are final up to rate * P - g; after END up to the true end
// rate * P) therefore keeps its carried rows in [0, lead - g) and receives this push's rows right after them.  Every conv
// runs "valid" over the window (output tau <-> time rate * P_old - g_out + tau), so a layer's input and output offsets
// are constants; only the per-slot row bounds vary, and they are built on the host once per push (TcProb::rb):
//   input rows before time 0 (rows standing for time before BEGIN) and past the rows available (or the true end) read
//   as zero; output rows past what is final are not written.
// One prep kernel per push moves each window's tail to its front (the rows the next push keeps), zeroes slots on BEGIN
// and copies the new mel frames in.
#include <algorithm>

#include "stream_common.cuh"

using namespace hgpk;

namespace {

constexpr int NRATE = 5;            // rate index 0: mel frames (mel, conv_pre out); 1 + i: output of up-sampling stage i
constexpr int NTEN = 2 + 4 * 19;    // windows per slot: mel, P0, then per stage X and T/Y of 3 chains x 3 pairs
constexpr int NCONV = 1 + 4 * 19;   // tensor-core convs per push: conv_pre, then per stage ups and 3 pairs x 2 convs

// ---- the layer table: lags, leads and lookahead, derived from the generator's hyper-parameters ----
struct Plan {
  int rate[NRATE];
  int lead[NRATE];
  int lag_p0;                       // conv_pre out
  int lag_in[4];                    // stage input (conv_pre out, or the mean of the previous stage's chains)
  int late[4];                      // ConvTranspose phases that read one input row ahead (the top ones, r >= u - late)
  int lag_x[4];                     // ConvTranspose out
  int lag_t[4][3][3], lag_y[4][3][3];   // [stage][chain j][pair m]
  int lag_m[4];                     // mean of the three chains of the stage
  int D;                            // lookahead in mel frames
};

constexpr int ups_e(int i, int r) {   // input shift of ConvTranspose phase r (see hifigan.cu repack_ups_kernel): -1 or 0
  return (r + (((vc::hg_upk(i) + vc::hg_rate(i) - 1) / 2 - r) % vc::hg_rate(i) + vc::hg_rate(i)) % vc::hg_rate(i) -
          (vc::hg_upk(i) + vc::hg_rate(i) - 1) / 2) / vc::hg_rate(i);
}

Plan make_plan() {
  Plan p{};
  p.rate[0] = 1;
  for (int i = 0; i < 4; ++i) p.rate[i + 1] = p.rate[i] * vc::hg_rate(i);
  // lags: a conv with half-width h needs h rows to its right; ConvTranspose phase r of input row tau reads rows
  // tau + e_r and tau + e_r + 1, so its output is final up to u * n_in - (phases reading row n_in)
  p.lag_p0 = 3;
  int lag = p.lag_p0;
  for (int i = 0; i < 4; ++i) {
    const int u = vc::hg_rate(i);
    p.late[i] = 0;
    for (int r = 0; r < u; ++r) p.late[i] += ups_e(i, r) == 0;
    p.lag_in[i] = lag;
    p.lag_x[i] = u * lag + p.late[i];
    p.lag_m[i] = 0;
    for (int j = 0; j < 3; ++j) {
      const int k = vc::hg_rbk(j);
      int g = p.lag_x[i];
      for (int m = 0; m < 3; ++m) {
        g += (k - 1) * vc::hg_dil(m) / 2;
        p.lag_t[i][j][m] = g;
        g += (k - 1) / 2;
        p.lag_y[i][j][m] = g;
      }
      p.lag_m[i] = std::max(p.lag_m[i], g);
    }
    lag = p.lag_m[i];
  }
  // conv_post (k = 7) adds 3 rows; output is emitted in whole frames
  p.D = (p.lag_m[3] + 3 + vc::HOP - 1) / vc::HOP;
  // leads: the oldest row any consumer of the rate reads in a push, relative to rate * P_old
  p.lead[0] = std::max(p.lag_p0 + 3, p.lag_p0 + 2);            // conv_pre reads mel from its first output - 3; ups 0 reads P0 from row - 2
  for (int i = 0; i < 4; ++i) {
    int need = i < 3 ? p.lag_m[i] + 2 : p.D * vc::HOP + 3;    // next ConvTranspose, or conv_post
    for (int j = 0; j < 3; ++j)
      for (int m = 0; m < 3; ++m) {
        const int k = vc::hg_rbk(j);
        need = std::max(need, p.lag_t[i][j][m] + (k - 1) * vc::hg_dil(m) / 2);
        need = std::max(need, p.lag_y[i][j][m] + (k - 1) / 2);
      }
    p.lead[i + 1] = need;
  }
  return p;
}

const Plan& plan() {
  static const Plan p = make_plan();
  return p;
}

struct StreamTen {
  float* p;
  int C, cap, keep, rate;   // keep = carried rows (lead - lag)
};

// per push, per slot: op bit0 zero the carried rows (BEGIN), bit1 move the tail of the last push to the front; shift =
// frames of that push; n = new mel frames to copy in
__global__ void __launch_bounds__(256) stream_prep_kernel(const StreamTen* __restrict__ tens, const int* __restrict__ tbl,
                                                          const float* __restrict__ mel, int F) {
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int op = tbl[3 * b], shift = tbl[3 * b + 1], n = tbl[3 * b + 2];
  if (op == 0 && (t != 0 || n == 0)) return;
  const StreamTen d = tens[t];
  float4* w = reinterpret_cast<float4*>(d.p + (size_t)b * d.cap * d.C);
  const int n4 = d.keep * d.C / 4;
  if (op & 1) {
    for (int i = tid; i < n4; i += 256) w[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  } else if (op & 2) {
    // rows [rate * shift, + keep) -> [0, keep): source and destination overlap when the push was shorter than the
    // carry, so each block of 1024 vectors is read completely before it is written, in ascending order
    const float4* src = w + (size_t)shift * d.rate * d.C / 4;
    constexpr int U = 4;
    for (int i0 = 0; i0 < n4; i0 += 256 * U) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * 256 + tid;
        if (i < n4) v[u] = src[i];
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * 256 + tid;
        if (i < n4) w[i] = v[u];
      }
      __syncthreads();
    }
  }
  if (t == 0 && n > 0) {   // the mel window: new frames after the carried ones
    const float4* src = reinterpret_cast<const float4*>(mel + (size_t)b * F * vc::MEL);
    for (int i = tid; i < n * vc::MEL / 4; i += 256) w[n4 + i] = src[i];
  }
}

// conv_post_kernel of hifigan.cu over a window: output sample o of slot b is window row p0 + o of the three chain
// outputs of the last stage; rows outside [lo, hi) are zero.  Same operations in the same order, so the same bits.
__global__ void __launch_bounds__(256) stream_post_kernel(const float* __restrict__ a0, const float* __restrict__ a1,
                                                          const float* __restrict__ a2, const float* __restrict__ w,
                                                          const float* __restrict__ bias, const int* __restrict__ tbl, int cap,
                                                          int wav_ld, float* __restrict__ wav) {
  constexpr int C = 32, KW = 7, TT = 256, ST = 33;
  __shared__ float xs[(TT + KW - 1) * ST];
  __shared__ float wsm[KW * C];
  const int b = blockIdx.y, t0 = blockIdx.x * TT, tid = threadIdx.x;
  const int lo = tbl[4 * b], hi = tbl[4 * b + 1], p0 = tbl[4 * b + 2], n = tbl[4 * b + 3];
  if (t0 >= n) return;
  if (tid < KW * C) wsm[tid] = w[tid];
  const size_t base = (size_t)b * cap * C;
  for (int e = tid; e < (TT + KW - 1) * (C / 4); e += 256) {
    int rr = e / (C / 4), q = e % (C / 4);
    int r = p0 + t0 - 3 + rr;
    float4 v = make_float4(0, 0, 0, 0);
    if (r >= lo && r < hi) {
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
    float* dd = xs + rr * ST + q * 4;
    dd[0] = v.x; dd[1] = v.y; dd[2] = v.z; dd[3] = v.w;
  }
  __syncthreads();
  const int t = t0 + tid;
  if (t >= n) return;
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < KW; ++j)
#pragma unroll
    for (int i = 0; i < C; ++i) acc = fmaf(xs[(tid + j) * ST + i], wsm[j * C + i], acc);
  wav[(size_t)b * wav_ld + t] = tanhf(acc + bias[0]);
}

// window index of the tensors: 0 mel, 1 P0, then per stage i: X, T[j][m], Y[j][m]
int ti_x(int i) { return 2 + 19 * i; }
int ti_t(int i, int j, int m) { return 2 + 19 * i + 1 + j * 3 + m; }
int ti_y(int i, int j, int m) { return 2 + 19 * i + 10 + j * 3 + m; }
// conv index: 0 conv_pre, then per stage i: ups, then pair m: conv1 of chains 0..2, conv2 of chains 0..2
int ci_ups(int i) { return 1 + 19 * i; }
int ci_rb(int i, int m, int which, int j) { return 1 + 19 * i + 1 + m * 6 + which * 3 + j; }

}  // namespace

// The shared slot state counts mel frames: received since BEGIN in P, emitted in E.
struct vtts_vocoder_stream : StreamBase {
  using StreamBase::StreamBase;
  int cap[NRATE] = {};
  StreamTen ten[NTEN];          // every window, then their device copy d_ten in the same allocation
  StreamTen* d_ten = nullptr;
  std::vector<int> tbl;         // host image of the per-push bounds table
};

int vtts_vocoder_stream_lookahead(void) { return plan().D; }

int vtts_vocoder_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_frames, vtts_vocoder_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "vocoder_stream_create", out, true, max_streams, max_chunk_frames, 4096, "max_chunk_frames");
  if (rc) return rc;
  if (!ctx->hg.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "vocoder_stream_create: hifigan weights not loaded");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const Plan& pl = plan();
  std::unique_ptr<vtts_vocoder_stream> vs(new vtts_vocoder_stream(ctx, max_streams, max_chunk_frames));
  for (int r = 0; r < NRATE; ++r) vs->cap[r] = pl.lead[r] + pl.rate[r] * max_chunk_frames;
  // window shapes: channels, rate index, lag
  auto shape = [&](int t, int C, int ri, int lag) { vs->ten[t] = StreamTen{nullptr, C, vs->cap[ri], pl.lead[ri] - lag, pl.rate[ri]}; };
  shape(0, vc::MEL, 0, 0);
  shape(1, vc::HG_C0, 0, pl.lag_p0);
  for (int i = 0, C = vc::HG_C0 / 2; i < 4; ++i, C /= 2) {
    shape(ti_x(i), C, i + 1, pl.lag_x[i]);
    for (int j = 0; j < 3; ++j)
      for (int m = 0; m < 3; ++m) {
        shape(ti_t(i, j, m), C, i + 1, pl.lag_t[i][j][m]);
        shape(ti_y(i, j, m), C, i + 1, pl.lag_y[i][j][m]);
      }
  }
  rc = stream_alloc(ctx, "vocoder_stream_create", *vs, [&](Arena& a) {
    for (int t = 0; t < NTEN; ++t) vs->ten[t].p = a.take<float>((size_t)max_streams * vs->ten[t].cap * vs->ten[t].C);
    vs->d_ten = a.take<StreamTen>(NTEN);
  });
  if (rc) return rc;
  VTTS_CUDA(cudaMemcpy(vs->d_ten, vs->ten, sizeof(vs->ten), cudaMemcpyHostToDevice));
  *out = vs.release();
  return VTTS_OK;
}

int vtts_vocoder_stream_destroy(vtts_ctx* ctx, vtts_vocoder_stream* vs) { return stream_destroy(ctx, "vocoder_stream_destroy", vs); }

int vtts_vocoder_stream_push(vtts_ctx* ctx, vtts_vocoder_stream* vs, const float* mel_dev, const int32_t* n_new, const uint8_t* flags,
                             float* wav_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "vocoder_stream_push", vs, mel_dev && n_new && flags && wav_dev && n_out);
  if (rc) return rc;
  if (!ctx->hg.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "vocoder_stream_push: hifigan weights not loaded");
  if (ctx->precision == VTTS_PRECISION_FP32)
    return ctx->fail(VTTS_ERR_BAD_ARG, "vocoder_stream_push: the strict fp32 mode has no streaming path; use bf16x3 or fp16");
  const int S = vs->S, F = vs->F;
  const Plan& pl = plan();
  const int D = pl.D, wav_ld = vc::HOP * (F + D);
  SlotState& sl = vs->slots;
  rc = sl.check(ctx, "vocoder_stream_push", F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;

  // ---- host bookkeeping: per slot the frames before and after this push; per conv and slot the row bounds ----
  std::vector<int> P0(S), act(S), end(S), nn(S);
  for (int s = 0; s < S; ++s) {
    act[s] = n_new[s] > 0 || flags[s] != 0;
    end[s] = (flags[s] & 2) != 0;
    nn[s] = n_new[s];
    P0[s] = (flags[s] & 1) ? 0 : (int)sl.P[s];
  }
  // table layout: [NCONV][S][3] conv bounds, [S][4] conv_post, [S][3] prep
  const size_t o_post = (size_t)NCONV * S * 3, o_prep = o_post + (size_t)S * 4, n_tbl = o_prep + (size_t)S * 3;
  vs->tbl.assign(n_tbl, 0);
  int* tb = vs->tbl.data();
  int tile_rows[NCONV];
  std::fill(tile_rows, tile_rows + NCONV, 1);   // every launch is issued every push (a fixed launch count); idle rows skip their tiles
  // ConvTranspose of stage i in block form (hifigan.cu hg_ups): block tau covers rows ups_out0(i) + u * tau .. + u - 1,
  // phases u/2.. of input row tau - 1 and ..u/2 - 1 of input row tau, and reads both.  Input row tau <-> input time
  // rate * P_old - lag_in - 1 + tau.  Block 0 also rewrites rows already final in the last push, from the same input
  // rows: same bits.
  auto ups_out0 = [&](int i) { return pl.lead[i + 1] - pl.lag_x[i] + pl.late[i] - vc::hg_rate(i) - vc::hg_rate(i) / 2; };
  auto ups_in_off = [&](int i) { return pl.lead[i] - pl.lag_in[i] - 2; };
  // conv c reads rate ri_in (inputs final up to lag_in) and writes rate ri_out with lag lag_out; its output tau <-> row
  // out0 + tau (ConvTranspose: the block of rows out0 + u * tau .. + u - 1)
  auto bounds = [&](int c, int ri_in, int lag_in, int ri_out, int lag_out, int u) {
    const int sin = pl.rate[ri_in], sout = pl.rate[ri_out];
    const int out0 = u > 1 ? ups_out0(ri_in) : pl.lead[ri_out] - lag_out;   // first row written by tau = 0
    for (int s = 0; s < S; ++s) {
      if (!act[s]) continue;
      int* r = tb + ((size_t)c * S + s) * 3;
      r[0] = std::max(0, pl.lead[ri_in] - sin * P0[s]);
      r[1] = sin * nn[s] + pl.lead[ri_in] - (end[s] ? 0 : lag_in);
      r[2] = sout * nn[s] + pl.lead[ri_out] - (end[s] ? 0 : lag_out);
      tile_rows[c] = std::max(tile_rows[c], (r[2] - out0 + u - 1) / u);
    }
  };
  bounds(0, 0, 0, 0, pl.lag_p0, 1);
  for (int i = 0; i < 4; ++i) {
    bounds(ci_ups(i), i, pl.lag_in[i], i + 1, pl.lag_x[i], vc::hg_rate(i));
    for (int m = 0; m < 3; ++m)
      for (int j = 0; j < 3; ++j) {
        bounds(ci_rb(i, m, 0, j), i + 1, m == 0 ? pl.lag_x[i] : pl.lag_y[i][j][m - 1], i + 1, pl.lag_t[i][j][m], 1);
        bounds(ci_rb(i, m, 1, j), i + 1, pl.lag_t[i][j][m], i + 1, pl.lag_y[i][j][m], 1);
      }
  }
  std::vector<int> emit(S, 0), P1(S);
  std::vector<long long> E1(S);
  int post_max = 0;
  for (int s = 0; s < S; ++s) {
    P1[s] = P0[s] + nn[s];
    const int e_old = (flags[s] & 1) ? 0 : (int)sl.E[s];
    const int e_new = !act[s] ? e_old : (end[s] ? P1[s] : std::max(e_old, P1[s] - D));
    emit[s] = e_new - e_old;
    E1[s] = e_new;
    if (act[s]) {
      const int L = pl.lead[4];
      int* r = tb + o_post + (size_t)s * 4;
      r[0] = std::max(0, L - vc::HOP * P0[s]);
      r[1] = vc::HOP * nn[s] + L - (end[s] ? 0 : pl.lag_m[3]);
      r[2] = vc::HOP * (e_old - P0[s]) + L;
      r[3] = vc::HOP * emit[s];
      post_max = std::max(post_max, r[3]);
    }
    int* q = tb + o_prep + (size_t)s * 3;
    if (flags[s] & 1) q[0] = 1;
    else if (act[s] && sl.pending[s] > 0) { q[0] = 2; q[1] = sl.pending[s]; }
    q[2] = nn[s];
  }

  // ---- device: one table copy, prep, conv_pre, four stages, conv_post ----
  rc = ctx->ensure_ws(n_tbl * sizeof(int) + 256);
  if (rc) return rc;
  int* dtb = reinterpret_cast<int*>(ctx->ws);
  // pageable source: the call returns once the table is staged, so vs->tbl may be rewritten by the next push
  VTTS_CUDA(cudaMemcpyAsync(dtb, tb, n_tbl * sizeof(int), cudaMemcpyHostToDevice, st));
  stream_prep_kernel<<<dim3(NTEN, S), 256, 0, st>>>(vs->d_ten, dtb + o_prep, mel_dev, F);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());

  const ModelWeights& M = ctx->hg;
  auto& W = M.t;
  const int f16 = ctx->precision == VTTS_PRECISION_FP16;
  const int pk = f16 ? PK_COUNT : 0;
  auto rb = [&](int c) { return dtb + (size_t)c * S * 3; };
  const auto& T = vs->ten;
  TcLaunch TL;
  // conv_pre: 80 -> 512, k7; tau <-> time P_old - 3 + tau reads mel rows from tau
  memset(&TL, 0, sizeof(TL));
  TL.nprob = 2; TL.Cin = vc::MEL; TL.N = 256; TL.in_ld = vc::MEL; TL.out_ld = vc::HG_C0;
  TL.B = S; TL.T_rows = vs->cap[0]; TL.rows_out = vs->cap[0]; TL.tile_rows = tile_rows[0]; TL.pre_mode = 0; TL.pre_slope = 1.f; TL.f16 = f16;
  for (int t = 0; t < 2; ++t) {
    TcProb& q = TL.p[t];
    q.x0 = T[0].p; q.wpk = M.tiles(pk + PK_PRE)[t]; q.bias = W[hgi::PRE_B] + 256 * t; q.out = T[1].p + 256 * t;
    q.k = 7; q.dil = 1; q.in_off = pl.lead[0] - pl.lag_p0 - 3; q.out_stride = 1; q.out_off = pl.lead[0] - pl.lag_p0; q.rb = rb(0);
  }
  if ((rc = vtts_launch_tc_conv(ctx, TL, st))) return rc;

  for (int i = 0, C = vc::HG_C0; i < 4; ++i, C /= 2) {
    const int u = vc::hg_rate(i), Co = C / 2;
    // ---- lrelu(0.1) [of the 3-way mean for i > 0] -> ConvTranspose as one conv over blocks of u output rows ----
    const int N = vtts_tc_tile_n(u * Co), nt = u * Co / N;
    memset(&TL, 0, sizeof(TL));
    TL.nprob = nt; TL.Cin = C; TL.N = N; TL.in_ld = C; TL.out_ld = u * Co; TL.out_sub = Co;
    TL.B = S; TL.T_rows = vs->cap[i]; TL.rows_out = vs->cap[i + 1]; TL.tile_rows = tile_rows[ci_ups(i)];
    TL.pre_mode = i == 0 ? 1 : 2; TL.pre_slope = 0.1f; TL.f16 = f16;
    for (int g = 0; g < nt; ++g) {
      TcProb& q = TL.p[g];
      if (i == 0) {
        q.x0 = T[1].p;
      } else {
        q.x0 = T[ti_y(i - 1, 0, 2)].p; q.x1 = T[ti_y(i - 1, 1, 2)].p; q.x2 = T[ti_y(i - 1, 2, 2)].p;
      }
      q.wpk = M.tiles(pk + PK_UPS(i))[g]; q.bias = M.d[D_UPS_BLK_B(i)] + g * N; q.out = T[ti_x(i)].p;
      q.k = 2; q.dil = 1; q.in_off = ups_in_off(i); q.out_stride = 1; q.out_off = 0; q.out_e0 = ups_out0(i) * Co + g * N;
      q.rb = rb(ci_ups(i));
    }
    if ((rc = vtts_launch_tc_conv(ctx, TL, st))) return rc;

    // ---- three ResBlock1 chains, each 3 x [lrelu, conv(d), lrelu, conv(1), + x] as two launches per pair ----
    for (int m = 0; m < 3; ++m) {
      const int d = vc::hg_dil(m);
      for (int which = 0; which < 2; ++which) {
        const int c0 = ci_rb(i, m, which, 0);
        memset(&TL, 0, sizeof(TL));
        TL.nprob = 3; TL.Cin = Co; TL.N = Co; TL.in_ld = Co; TL.out_ld = Co;
        TL.B = S; TL.T_rows = vs->cap[i + 1]; TL.rows_out = vs->cap[i + 1];
        TL.pre_mode = 1; TL.pre_slope = 0.1f; TL.f16 = f16;
        for (int j = 0; j < 3; ++j) {
          const int kk = vc::hg_rbk(j), n = i * 3 + j, c = c0 + j;
          const int dd = which == 0 ? d : 1, h = (kk - 1) * dd / 2;
          const int lag_out = which == 0 ? pl.lag_t[i][j][m] : pl.lag_y[i][j][m];
          const float* x = m == 0 ? T[ti_x(i)].p : T[ti_y(i, j, m - 1)].p;
          TcProb& q = TL.p[j];
          q.x0 = which == 0 ? x : T[ti_t(i, j, m)].p;
          q.wpk = M.tiles(pk + PK_RB(n, which, m))[0];
          q.bias = W[hgi::RB_B(n, which, m)];
          q.resid = which == 0 ? nullptr : x;   // same window row as the output: x at the pair output's time
          q.out = which == 0 ? T[ti_t(i, j, m)].p : T[ti_y(i, j, m)].p;
          q.k = kk; q.dil = dd; q.in_off = pl.lead[i + 1] - lag_out - h; q.out_stride = 1; q.out_off = pl.lead[i + 1] - lag_out;
          q.rb = rb(c);
          TL.tile_rows = std::max(TL.tile_rows, tile_rows[c]);
        }
        if ((rc = vtts_launch_tc_conv(ctx, TL, st))) return rc;
      }
    }
  }
  {
    dim3 grid(std::max(1, (post_max + 255) / 256), S);
    stream_post_kernel<<<grid, 256, 0, st>>>(T[ti_y(3, 0, 2)].p, T[ti_y(3, 1, 2)].p, T[ti_y(3, 2, 2)].p, W[hgi::POST_W], W[hgi::POST_B],
                                             dtb + o_post, vs->cap[4], wav_ld, wav_dev);
    ctx->launches++;
    VTTS_CUDA(cudaGetLastError());
  }

  for (int s = 0; s < S; ++s) n_out[s] = emit[s];
  sl.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_vocoder_stream_push_host(vtts_ctx* ctx, vtts_vocoder_stream* vs, const float* mel, const int32_t* n_new, const uint8_t* flags,
                                  float* wav, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "vocoder_stream_push_host", vs, mel && wav);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(mel, (size_t)vs->S * vs->F * vc::MEL * 4), o_y = hs.out((size_t)vs->S * vc::HOP * (vs->F + plan().D) * 4, wav);
  return hs.run([&](cudaStream_t st) {
    return vtts_vocoder_stream_push(ctx, vs, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, st);
  });
}
