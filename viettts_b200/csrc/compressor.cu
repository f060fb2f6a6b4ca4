// Feed-forward compressor of one mono row, fp32 on the device in every vtts_precision mode (oracle/compressor_oracle.py
// states it in float64):
//   L = 20 log10 |x|;  x_L = L - G(L), G the soft-knee gain computer (threshold T, ratio R, knee W; exactly 0 below the
//   knee and at L = -inf);  release y1[t] = max(x_L[t], a_R y1[t - 1] + b_R x_L[t]);  attack
//   y_L[t] = a_A y_L[t - 1] + b_A y1[t] (both from 0);  y = (x m) 10^(-y_L / 20);  reduction = -max y_L.
// a = fp32(exp(-1000 / (tau rate))) and b = 1 - a, exact in fp32 (a >= 0.78 over the parameter ranges), so each stage's
// DC gain b / (1 - a) is 1 to fp32 precision.
//
// Invariant (as in limiter.cu).  Both stages scan as maps over blocks of Q = 256 samples fixed by absolute index.  The
// release steps are the limiter's monotone maps (Map, map_fold, map_apply in vtts_internal.cuh) with a = x_L[t]; the
// attack steps are the affine maps d -> fma(a_A, d, b_A y1[t]), held as Maps with c = -inf (map_apply is then exactly
// the affine map), composing as (m, k) -> (a_A m, fma(a_A, k, b_A y1)).  Per stage: a fold kernel (one thread per
// (row, block)) folds the block's maps in sample order, a chain kernel (one thread per row) walks the block maps from 0
// (or the carried value) to each block's entering value, and the next kernel refolds the block from it.  x_L is
// recomputed from x in every pass.  A row therefore gives the same bits alone, in any batch position, in every
// precision mode, and through the stream at any push pattern.  Rows below the knee (and R = 1) have y_L = 0 everywhere
// and come back as x m bit for bit.
//
// Stream.  No lookahead: every push releases the samples it brings, read where they are (no window).  Per slot the
// partial release and attack maps of the block holding its next sample, that block's y1 and y_L entering values, and
// the running maximum of y_L.  Every push issues the same six launches after its one table copy.
#include "compressor_kernels.cuh"

using namespace cpk;

namespace {

// the parameters and batch shape of a one-shot call of entry point `who`
int cp_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, float threshold_db, float ratio, float knee_db, float attack_ms,
            float release_ms, float makeup_db, CpParams* p) {
  const int rc = cp_params(ctx, who, rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, p);
  return rc ? rc : batch_check(ctx, who, B, S, S_MAX);
}

int cp_launch(vtts_ctx* ctx, const CpParams& p, const float* x, const int32_t* n_in, int B, int S, float* y, float* reduction_db, cudaStream_t st) {
  const int rc = ctx->ensure_ws(cp_oneshot_bytes(B, S));
  if (rc) return rc;
  CpBufs w{};
  Arena a(ctx->ws, SIZE_MAX, false);
  cp_carve(a, B, cp_blocks_max(S), &w);
  return cp_run(ctx, p, x, S, S, n_in, nullptr, B, S, S, w, y, S, reduction_db, st);
}

}  // namespace

int vtts_compress(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float threshold_db, float ratio,
                  float knee_db, float attack_ms, float release_ms, float makeup_db, float* y_dev, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  CpParams p;
  const int rc = cp_args(ctx, "compress", B, S, rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, &p);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "compress: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return cp_launch(ctx, p, x_dev, n_dev, B, S, y_dev, reduction_db_dev, (cudaStream_t)stream);
}

int vtts_compress_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float threshold_db, float ratio,
                       float knee_db, float attack_ms, float release_ms, float makeup_db, float* y, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  CpParams p;
  int rc = cp_args(ctx, "compress_host", B, S, rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, &p);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("compress_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_r = hs.out((size_t)B * 4, reduction_db), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return cp_launch(ctx, p, hs.x(), hs.n(), B, S, hs.dev<float>(o_y), hs.dev<float>(o_r), st); });
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and released in E (the same: no lookahead).  A push reads x_dev
// and writes y_dev in place of a window: slot s's new samples [P0, P1) sit at x_dev[s][0, n_new[s]).
struct vtts_compressor_stream : SampleStream<CpRow> {
  using SampleStream::SampleStream;
  CpParams p{};
  CpBufs w{};
};

int vtts_compressor_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float threshold_db, float ratio,
                                  float knee_db, float attack_ms, float release_ms, float makeup_db, vtts_compressor_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "compressor_stream_create", out, true, max_streams, max_chunk_samples);
  if (rc) return rc;
  CpParams p;
  rc = cp_params(ctx, "compressor_stream_create", rate, threshold_db, ratio, knee_db, attack_ms, release_ms, makeup_db, &p);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_compressor_stream> cs(new vtts_compressor_stream(ctx, max_streams, max_chunk_samples, 0));
  cs->p = p;
  const size_t S = max_streams;
  rc = stream_alloc(ctx, "compressor_stream_create", *cs, [&](Arena& a) {
    cp_carve(a, S, cp_blocks_max(max_chunk_samples), &cs->w);
    cs->w.carry_r = a.take<float4>(S);
    cs->w.carry_a = a.take<float4>(S);
    cs->w.carry_y1 = a.take<float>(S);
    cs->w.carry_yl = a.take<float>(S);
    cs->w.carry_max = a.take<float>(S);
    cs->carve_tables(a);
  });
  if (rc) return rc;
  *out = cs.release();
  return VTTS_OK;
}

int vtts_compressor_stream_destroy(vtts_ctx* ctx, vtts_compressor_stream* cs) { return stream_destroy(ctx, "compressor_stream_destroy", cs); }

int vtts_compressor_stream_push(vtts_ctx* ctx, vtts_compressor_stream* cs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "compressor_stream_push", cs, x_dev && n_new && flags && y_dev && n_out && reduction_db_dev);
  if (rc) return rc;
  const SlotState& sl = cs->slots;
  rc = sl.check(ctx, "compressor_stream_push", cs->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = cs->S;

  // ---- host bookkeeping: every sample is released in the push that brings it ----
  CpRow* rows = cs->rows<0>();
  std::vector<long long> E1(S);
  long long max_rn = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    const CpRow r = cp_stream_row(P0, P1, begin);
    rows[s] = r;
    E1[s] = P1;
    n_out[s] = (int32_t)(P1 - P0);
    max_rn = std::max(max_rn, r.rn);
  }

  // ---- device: one table copy, then the compressor's six launches ----
  rc = cs->upload_rows(st);
  if (rc) return rc;
  rc = cp_run(ctx, cs->p, x_dev, cs->F, cs->F, nullptr, cs->d_rows<0>(), S, max_rn, max_rn, cs->w, y_dev, cs->F, reduction_db_dev, st);
  if (rc) return rc;
  cs->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_compressor_stream_push_host(vtts_ctx* ctx, vtts_compressor_stream* cs, const float* x, const int32_t* n_new, const uint8_t* flags,
                                     float* y, int32_t* n_out, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "compressor_stream_push_host", cs, x && y && reduction_db);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)cs->S * cs->F * 4), o_y = hs.out((size_t)cs->S * cs->F * 4, y), o_r = hs.out((size_t)cs->S * 4, reduction_db);
  return hs.run([&](cudaStream_t st) {
    return vtts_compressor_stream_push(ctx, cs, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, hs.dev<float>(o_r), st);
  });
}
