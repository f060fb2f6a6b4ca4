// Streaming acoustic model: every open slot advances its autoregressive decoder a few frames per push, and the mel frames
// whose postnet receptive field is complete are emitted.  A slot's emitted frames, concatenated, are bit-identical to
// vtts_acoustic_forward of that utterance alone (same precision and dropout mode).
//
// begin  runs the acoustic front half (TokenEncoder, upsample, hoisted cond projections) of the new rows with the
//        one-shot code and keeps each row's zc0 / zc1 in its slot, with zero carried state.
// push   one launch of decoder_scan_kernel<true> over the open slots (each continues from its own absolute frame), the
//        output projection of the new frames into the slot's melpre, then the postnet over a per-slot window
//        [max(0, a - D), p) of melpre (a = first frame not emitted, p = frames scanned).  The five k = 5 convs of the
//        postnet reach D = 10 frames to each side, so window frames in [a, p - D) -- or up to the true end once the
//        slot has scanned everything -- see exactly the inputs they see in the one-shot postnet; the conv dispatcher
//        sums each output element in a fixed order whatever the window length, so they get the same bits.
#include <algorithm>

#include "stream_common.cuh"

namespace {

constexpr int D_A = 10;           // postnet lookahead: five k = 5 convs, 2 frames each
constexpr int MAX_SLOTS = 128;    // one scan launch holds 128 rows
constexpr int ZW = 4 * vc::DEC_H; // 2048 columns of zc0 / zc1

// per launch row: slot, t0 (first frame scanned now), n (frames scanned now), w0 (first window frame), W (window
// frames, 0 = no postnet this push), off (window index of the first frame emitted), cnt (frames emitted)
enum { R_SLOT, R_T0, R_N, R_W0, R_W, R_OFF, R_CNT, R_STRIDE };

// win[r][j] = melpre of slot frame w0 + j: frames before t0 come from the slot's melpre, the new ones from this push's
// projection, which is also stored into the slot's melpre.  One block per (row, 16-frame chunk).
__global__ void __launch_bounds__(256) stream_window_kernel(const int* __restrict__ tbl, const float* __restrict__ proj, int F,
                                                            float* __restrict__ melpre, int NF, float* __restrict__ win, int WM) {
  const int r = blockIdx.y, tid = threadIdx.x;
  const int* q = tbl + r * R_STRIDE;
  const int slot = q[R_SLOT], t0 = q[R_T0], n = q[R_N], w0 = q[R_W0], W = q[R_W];
  constexpr int V = vc::MEL / 4;
  float4* mp = reinterpret_cast<float4*>(melpre + (size_t)slot * NF * vc::MEL);
  const float4* pp = reinterpret_cast<const float4*>(proj + (size_t)r * F * vc::MEL);
  const int f0 = blockIdx.x * 16;
  for (int e = tid; e < 16 * V; e += 256) {
    const int i = f0 + e / V, v = e % V;
    if (i < n) mp[(size_t)(t0 + i) * V + v] = pp[(size_t)i * V + v];
  }
  float4* wp = reinterpret_cast<float4*>(win + (size_t)r * WM * vc::MEL);
  for (int e = tid; e < 16 * V; e += 256) {
    const int j = f0 + e / V, v = e % V, f = w0 + j;
    if (j < W) wp[(size_t)j * V + v] = f < t0 ? mp[(size_t)f * V + v] : pp[(size_t)(f - t0) * V + v];
  }
}

// mel[slot][k] = post[r][off + k], k < cnt
__global__ void __launch_bounds__(256) stream_emit_kernel(const int* __restrict__ tbl, const float* __restrict__ post, int WM,
                                                          float* __restrict__ mel, int OF) {
  const int r = blockIdx.y, tid = threadIdx.x;
  const int* q = tbl + r * R_STRIDE;
  const int slot = q[R_SLOT], off = q[R_OFF], cnt = q[R_CNT];
  constexpr int V = vc::MEL / 4;
  const float4* src = reinterpret_cast<const float4*>(post + ((size_t)r * WM + off) * vc::MEL);
  float4* dst = reinterpret_cast<float4*>(mel + (size_t)slot * OF * vc::MEL);
  for (int e = blockIdx.x * 256 + tid; e < cnt * V; e += gridDim.x * 256) dst[e] = src[e];
}

}  // namespace

struct vtts_acoustic_stream {
  vtts_ctx* ctx = nullptr;
  int S = 0, F = 0, NF = 0, LT = 0, WM = 0;   // slots, max chunk frames, max frames, max tokens, window rows F + 2 D
  int mode = 0;
  uint64_t seed = 0;
  void* mem = nullptr;
  float *zc0 = nullptr, *zc1 = nullptr, *melpre = nullptr, *state = nullptr;
  uint8_t* keep = nullptr;
  uint2* subkeys = nullptr;
  float *hout = nullptr, *proj = nullptr, *win = nullptr, *q0 = nullptr, *q1 = nullptr, *post = nullptr;
  float *p1 = nullptr, *p2 = nullptr, *h0 = nullptr, *h1 = nullptr;
  unsigned int* bar = nullptr;
  int4* rows = nullptr;     // device [MAX_SLOTS] scan rows
  int* tbl = nullptr;       // device [MAX_SLOTS][R_STRIDE], then lens
  int* lens = nullptr;      // device [2][MAX_SLOTS]: projection rows (n), postnet rows (W)
  // host state per slot: open, frames scanned, frames emitted, frames to scan, frames to emit
  std::vector<int> open, P, E, P_end, n_emit;
  std::vector<int> h_tbl;   // host image of rows | tbl | lens
};

extern "C" {

int vtts_acoustic_stream_lookahead(void) { return D_A; }

int vtts_acoustic_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_frames, int max_frames, int max_tokens, int dropout_mode,
                                uint64_t seed, vtts_acoustic_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "acoustic_stream_create", out, true, max_streams, max_chunk_frames, 4096, "max_chunk_frames", MAX_SLOTS);
  if (rc) return rc;
  if (!ctx->ac.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "acoustic_stream_create: acoustic weights not loaded");
  if (max_frames < 1 || max_frames > (1 << 24) || max_tokens < 1 || max_tokens > vtts_acoustic_max_tokens())
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_create: max_frames=%d max_tokens=%d (1..%d, 1..%d)", max_frames, max_tokens, 1 << 24,
                     vtts_acoustic_max_tokens());
  if (dropout_mode < VTTS_DROPOUT_OFF || dropout_mode > VTTS_DROPOUT_REFERENCE)
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_create: dropout_mode %d", dropout_mode);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  vtts_acoustic_stream* as = new vtts_acoustic_stream;
  as->ctx = ctx;
  as->S = max_streams; as->F = max_chunk_frames; as->NF = max_frames; as->LT = max_tokens;
  as->WM = max_chunk_frames + 2 * D_A;
  as->mode = dropout_mode; as->seed = seed;
  const size_t S = max_streams, F = max_chunk_frames, NF = max_frames, WM = as->WM;
  Arena sz(nullptr, 0, true);
  auto carve = [&](Arena& ar) {
    as->zc0 = ar.take<float>(S * NF * ZW);
    as->zc1 = ar.take<float>(S * NF * ZW);
    as->melpre = ar.take<float>(S * NF * vc::MEL);
    as->state = ar.take<float>(S * 4 * vc::DEC_H);
    as->keep = ar.take<uint8_t>(dropout_mode == VTTS_DROPOUT_MASK ? S * NF * 2 * vc::PRENET : 0);
    as->subkeys = ar.take<uint2>(dropout_mode == VTTS_DROPOUT_REFERENCE ? 2 * NF : 0);
    as->hout = ar.take<float>(S * F * 2 * vc::DEC_H);
    as->proj = ar.take<float>(S * F * vc::MEL);
    as->win = ar.take<float>(S * WM * vc::MEL);
    as->q0 = ar.take<float>(S * WM * vc::POSTNET);
    as->q1 = ar.take<float>(S * WM * vc::POSTNET);
    as->post = ar.take<float>(S * WM * vc::MEL);
    as->p1 = ar.take<float>((size_t)MAX_SLOTS * vc::PRENET);
    as->p2 = ar.take<float>((size_t)MAX_SLOTS * vc::PRENET);
    as->h0 = ar.take<float>((size_t)2 * MAX_SLOTS * vc::DEC_H);
    as->h1 = ar.take<float>((size_t)2 * MAX_SLOTS * vc::DEC_H);
    as->bar = ar.take<unsigned int>(64);
    as->rows = ar.take<int4>(MAX_SLOTS);
    as->tbl = ar.take<int>((size_t)MAX_SLOTS * R_STRIDE + 2 * MAX_SLOTS);   // lens follow the table: one copy per push
    as->lens = ar.measure ? nullptr : as->tbl + (size_t)MAX_SLOTS * R_STRIDE;
  };
  carve(sz);
  const size_t bytes = sz.off + 256;
  cudaError_t e = cudaMalloc(&as->mem, bytes);
  if (e == cudaSuccess) e = cudaMemset(as->mem, 0, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (as->mem) cudaFree(as->mem);
    delete as;
    return ctx->fail(e == cudaErrorMemoryAllocation ? VTTS_ERR_OOM : VTTS_ERR_CUDA, "acoustic_stream_create: %zu bytes: %s", bytes,
                     cudaGetErrorString(e));
  }
  Arena ar(as->mem, bytes, false);
  carve(ar);
  if (dropout_mode == VTTS_DROPOUT_REFERENCE) {
    // frame t, prenet layer l of every slot draws with sub-key 2t + l of the checkpoint key's chain
    rc = vtts_ref_subkeys(ctx, seed, 2 * max_frames, as->subkeys, nullptr);
    if (rc == VTTS_OK && cudaDeviceSynchronize() != cudaSuccess) rc = ctx->fail(VTTS_ERR_CUDA, "acoustic_stream_create: sub-key chain failed");
    if (rc) {
      cudaFree(as->mem);
      delete as;
      return rc;
    }
  }
  as->open.assign(max_streams, 0);
  as->P.assign(max_streams, 0);
  as->E.assign(max_streams, 0);
  as->P_end.assign(max_streams, 0);
  as->n_emit.assign(max_streams, 0);
  *out = as;
  return VTTS_OK;
}

int vtts_acoustic_stream_destroy(vtts_ctx* ctx, vtts_acoustic_stream* as) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!as) return VTTS_OK;
  if (as->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_destroy: the stream belongs to another context");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());   // a push may still be running on the caller's stream
  if (ctx->tap_melpre == as->melpre) ctx->clear_taps();
  cudaFree(as->mem);
  delete as;
  return VTTS_OK;
}

int vtts_acoustic_stream_begin(vtts_ctx* ctx, vtts_acoustic_stream* as, int nb, const int32_t* slots, const int32_t* tokens,
                               const int32_t* lengths, const float* dur_frames, const int32_t* n_frames, const int32_t* n_emit,
                               const uint8_t* keep, int L) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!as || as->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: the stream belongs to another context");
  if (!slots || !tokens || !dur_frames || !n_frames) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: null pointer");
  if (nb < 1 || nb > as->S || L < 1 || L > as->LT)
    return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: nb=%d L=%d (1..%d rows, 1..%d tokens)", nb, L, as->S, as->LT);
  if (as->mode == VTTS_DROPOUT_MASK && !keep) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: dropout_mode MASK needs keep");
  int N = 0;
  std::vector<int> seen(as->S, 0);
  for (int i = 0; i < nb; ++i) {
    const int s = slots[i];
    if (s < 0 || s >= as->S) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: slot %d outside [0, %d)", s, as->S);
    if (seen[s]++) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: slot %d given twice", s);
    if (as->open[s]) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: slot %d is still open", s);
    if (n_frames[i] < 1 || n_frames[i] > as->NF)
      return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: n_frames[%d]=%d outside [1, max_frames=%d]", i, n_frames[i], as->NF);
    const int ne = n_emit ? n_emit[i] : n_frames[i];
    if (ne < 1 || ne > n_frames[i]) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: n_emit[%d]=%d outside [1, %d]", i, ne, n_frames[i]);
    if (lengths && (lengths[i] < 1 || lengths[i] > L))
      return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_begin: lengths[%d]=%d outside [1, %d]", i, lengths[i], L);
    N = std::max(N, n_frames[i]);
  }
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());   // earlier pushes may still read the slots' memory
  // ---- stage the rows, run the one-shot front half, keep each row's zc0 / zc1 in its slot ----
  int rc = ctx->ensure_ws(vtts_acoustic_ws_bytes(nb, L, N));
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_tok = hs.in(tokens, (size_t)nb * L * 4), o_len = hs.in(lengths, (size_t)nb * 4);
  const size_t o_dur = hs.in(dur_frames, (size_t)nb * L * 4), o_nf = hs.in(n_frames, (size_t)nb * 4);
  rc = hs.upload();
  if (rc) return rc;
  cudaStream_t st = hs.st;
  const float *zc0 = nullptr, *zc1 = nullptr;
  rc = vtts_acoustic_front(ctx, hs.dev<const int32_t>(o_tok), lengths ? hs.dev<const int32_t>(o_len) : nullptr, hs.dev<const float>(o_dur),
                           hs.dev<const int32_t>(o_nf), nb, L, N, &zc0, &zc1, st);
  if (rc) return rc;
  std::vector<int> pend(nb);
  for (int i = 0; i < nb; ++i) {
    const int s = slots[i], ne = n_emit ? n_emit[i] : n_frames[i];
    // frames before n_emit never see later ones, and frame n_emit - 1 sees D frames past it
    pend[i] = std::min(n_frames[i], ne + D_A);
    const size_t zb = (size_t)pend[i] * ZW * sizeof(float);
    VTTS_CUDA(cudaMemcpyAsync(as->zc0 + (size_t)s * as->NF * ZW, zc0 + (size_t)i * N * ZW, zb, cudaMemcpyDeviceToDevice, st));
    VTTS_CUDA(cudaMemcpyAsync(as->zc1 + (size_t)s * as->NF * ZW, zc1 + (size_t)i * N * ZW, zb, cudaMemcpyDeviceToDevice, st));
    VTTS_CUDA(cudaMemsetAsync(as->state + (size_t)s * 4 * vc::DEC_H, 0, 4 * vc::DEC_H * sizeof(float), st));
    if (as->mode == VTTS_DROPOUT_MASK)   // keep [nb][N][2][256] (host)
      VTTS_CUDA(cudaMemcpyAsync(as->keep + (size_t)s * as->NF * 2 * vc::PRENET, keep + (size_t)i * N * 2 * vc::PRENET,
                                (size_t)pend[i] * 2 * vc::PRENET, cudaMemcpyHostToDevice, st));
  }
  rc = hs.finish();
  if (rc) return rc;
  for (int i = 0; i < nb; ++i) {
    const int s = slots[i];
    as->open[s] = 1;
    as->P[s] = 0;
    as->E[s] = 0;
    as->P_end[s] = pend[i];
    as->n_emit[s] = n_emit ? n_emit[i] : n_frames[i];
  }
  return VTTS_OK;
}

int vtts_acoustic_stream_push(vtts_ctx* ctx, vtts_acoustic_stream* as, float* mel_dev, int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!as || as->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_push: the stream belongs to another context");
  if (!mel_dev || !n_out) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_push: null pointer");
  if (!ctx->ac.loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "acoustic_stream_push: acoustic weights not loaded");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = as->S, F = as->F;
  // ---- host schedule, fixed before anything is launched ----
  as->h_tbl.assign((size_t)MAX_SLOTS * 4 + (size_t)MAX_SLOTS * R_STRIDE + 2 * MAX_SLOTS, 0);
  int* hrows = as->h_tbl.data();
  int* htbl = hrows + MAX_SLOTS * 4;
  int* hlen = htbl + MAX_SLOTS * R_STRIDE;
  int nb = 0, nmax = 0;
  std::vector<int> P1(S), E1(S);
  for (int s = 0; s < S; ++s) {
    n_out[s] = 0;
    if (!as->open[s]) continue;
    const int t0 = as->P[s], n = std::min(F, as->P_end[s] - t0), p = t0 + n, a = as->E[s];
    const int e = p == as->P_end[s] ? as->n_emit[s] : std::min(as->n_emit[s], std::max(0, p - D_A));
    const int cnt = e - a, w0 = std::max(0, a - D_A);
    int* q = htbl + nb * R_STRIDE;
    q[R_SLOT] = s; q[R_T0] = t0; q[R_N] = n; q[R_W0] = w0; q[R_W] = cnt > 0 ? p - w0 : 0; q[R_OFF] = a - w0; q[R_CNT] = cnt;
    hrows[nb * 4 + 0] = s; hrows[nb * 4 + 1] = t0; hrows[nb * 4 + 2] = n;
    hlen[nb] = n;
    hlen[MAX_SLOTS + nb] = q[R_W];
    P1[s] = p;
    E1[s] = e;
    n_out[s] = cnt;
    nmax = std::max(nmax, n);
    ++nb;
  }
  if (nb == 0) return VTTS_OK;
  // ---- device: one table copy, the scan, projection, window, postnet, emit ----
  // pageable source: the call returns once the table is staged, so h_tbl may be rewritten by the next push
  static_assert(sizeof(int4) == 4 * sizeof(int), "int4 row table");
  VTTS_CUDA(cudaMemcpyAsync(as->rows, hrows, (size_t)MAX_SLOTS * 4 * sizeof(int), cudaMemcpyHostToDevice, st));
  VTTS_CUDA(cudaMemcpyAsync(as->tbl, htbl, ((size_t)MAX_SLOTS * R_STRIDE + 2 * MAX_SLOTS) * sizeof(int), cudaMemcpyHostToDevice, st));
  DecResume r;
  r.zc0 = as->zc0; r.zc1 = as->zc1; r.keep = as->keep; r.subkeys = as->subkeys; r.seed = as->seed; r.mode = as->mode;
  r.rows = as->rows; r.B = nb; r.nmax = nmax; r.state = as->state; r.zstride = as->NF; r.hstride = F;
  r.p1 = as->p1; r.p2 = as->p2; r.h0 = as->h0; r.h1 = as->h1; r.hout = as->hout; r.bar = as->bar;
  int rc = vtts_decoder_scan_resume(ctx, r, st);
  if (rc) return rc;
  rc = vtts_acoustic_project(ctx, as->hout, as->lens, nb, F, as->proj, st);
  if (rc) return rc;
  stream_window_kernel<<<dim3((as->WM + 15) / 16, nb), 256, 0, st>>>(as->tbl, as->proj, F, as->melpre, as->NF, as->win, as->WM);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  rc = vtts_acoustic_postnet(ctx, as->win, as->lens + MAX_SLOTS, nb, as->WM, as->q0, as->q1, as->post, st);
  if (rc) return rc;
  stream_emit_kernel<<<dim3(4, nb), 256, 0, st>>>(as->tbl, as->post, as->WM, mel_dev, F + D_A);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  // the stream's projection outputs so far are the mel_pre tap of this push ([S][max_frames][80])
  ctx->clear_taps();
  ctx->tap_melpre = as->melpre;
  ctx->tap_melpre_n = (int64_t)S * as->NF * vc::MEL;
  // ---- commit ----
  for (int s = 0; s < S; ++s) {
    if (!as->open[s]) continue;
    as->P[s] = P1[s];
    as->E[s] = E1[s];
    if (P1[s] == as->P_end[s]) as->open[s] = 0;
  }
  return VTTS_OK;
}

int vtts_acoustic_stream_push_host(vtts_ctx* ctx, vtts_acoustic_stream* as, float* mel, int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!as || as->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_push_host: the stream belongs to another context");
  if (!mel || !n_out) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_stream_push_host: null pointer");
  const size_t row_b = (size_t)(as->F + D_A) * vc::MEL * sizeof(float);
  HostStage hs(ctx);
  const size_t o_mel = hs.out((size_t)as->S * row_b);
  return hs.run([&](cudaStream_t st) {
    int rc = vtts_acoustic_stream_push(ctx, as, hs.dev<float>(o_mel), n_out, st);
    // only the rows that received frames are copied back
    for (int s = 0; s < as->S && !rc; ++s)
      if (n_out[s]) rc = hs.fetch(o_mel + s * row_b, (char*)mel + s * row_b, (size_t)n_out[s] * vc::MEL * sizeof(float));
    return rc;
  });
}

}  // extern "C"
