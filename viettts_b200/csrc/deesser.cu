// Split-band de-esser of one mono row, fp32 on the device in every vtts_precision mode (oracle/deesser_oracle.py states
// it in float64):
//   h = the second-order Butterworth high-pass at the crossover over x (the equalizer's one section, from zero state);
//   y_L = the compressor's detector (gain computer, release, attack) on L = 20 log10 |h|, no makeup;
//   y^_L = min(y_L, range);  y = x - (1 - g) h, g = 10^(-y^_L / 20);  reduction = -max y^_L.
// The band below the crossover, x - h, passes untouched; the high band is scaled by g only while it is loud.
//
// Composition.  The sidechain is the equalizer's block and chain kernels (eq_kernels.cuh) writing h into workspace; the
// detector is the compressor's fold, chain and finish kernels (compressor_kernels.cuh) reading h as their level source,
// and its apply kernel with the split output rule CpSplit: y = fmaf(g - 1, h, x) where y^_L > 0, x itself where y^_L = 0,
// so rows whose high band stays below the knee (and ratio 1, and range 0) come back as x bit for bit.  Both invariants
// hold unchanged (1024-sample filter blocks, 256-sample detector blocks, fixed by absolute sample index), so a row gives
// the same bits alone, in any batch position, in every precision mode and through the stream at any push pattern.
//
// Stream.  No lookahead: every push releases the samples it brings.  Per slot the equalizer stream's state (a window
// of the incomplete block's samples, the filter state at that block's start) and the compressor stream's (partial maps,
// entering values, largest y^_L).  h of the push's new samples lands in a [S][F] buffer laid out as x, which the
// detector reads beside x.  Every push issues one table copy and the same ten launches: the window step, the
// equalizer's three, the compressor's six.
#include "compressor_kernels.cuh"
#include "eq_kernels.cuh"

namespace {

struct DsParams {
  eqk::EqFilter f;   // the crossover high-pass
  cpk::CpParams p;   // the detector (makeup factor 1)
  float range;       // the cap on y_L, dB
};

int ds_params(vtts_ctx* ctx, const char* who, int rate, float freq_hz, float threshold_db, float ratio, float knee_db, float attack_ms,
              float release_ms, float range_db, DsParams* d) {
  int rc = cpk::cp_params(ctx, who, rate, threshold_db, ratio, knee_db, attack_ms, release_ms, 0.f, &d->p);
  if (rc) return rc;
  if (!((double)freq_hz >= 1000.0 && (double)freq_hz <= 0.45 * rate))
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: freq %g Hz (in [1000, 0.45 rate = %g])", who, (double)freq_hz, 0.45 * rate);
  if (!(range_db >= 0.f && range_db <= 24.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: range %g dB (in [0, 24])", who, (double)range_db);
  double sos[6];
  int K = 0;
  if (vtts_eq_design(VTTS_EQ_HIGHPASS, rate, freq_hz, 0.0, 0.0, 2, sos, &K) != VTTS_OK)
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: no high-pass at freq %g Hz", who, (double)freq_hz);
  d->range = range_db;
  return eqk::eq_filter(ctx, who, sos, K, &d->f);
}

// the one-shot workspace: h [B][S], the equalizer's block end and entering states, the compressor's buffers
struct DsBufs {
  float *h, *e, *s;
  cpk::CpBufs w;
};

void ds_carve(Arena& a, int B, int S, DsBufs* d) {
  const int nb = (S + eqk::Q - 1) / eqk::Q;
  d->h = a.take<float>((size_t)B * S);
  d->e = a.take<float>((size_t)B * nb * eqk::NS);
  d->s = a.take<float>((size_t)B * nb * eqk::NS);
  d->w = cpk::CpBufs{};
  cpk::cp_carve(a, B, cpk::cp_blocks_max(S), &d->w);
}

// the parameters and batch shape of a one-shot call of entry point `who`
int ds_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, float freq_hz, float threshold_db, float ratio, float knee_db,
            float attack_ms, float release_ms, float range_db, DsParams* d) {
  const int rc = ds_params(ctx, who, rate, freq_hz, threshold_db, ratio, knee_db, attack_ms, release_ms, range_db, d);
  return rc ? rc : batch_check(ctx, who, B, S, cpk::S_MAX);
}

int ds_launch(vtts_ctx* ctx, const DsParams& d, const float* x, const int32_t* n_in, int B, int S, float* y, float* reduction_db, cudaStream_t st) {
  Arena m(nullptr, 0, true);
  DsBufs w;
  ds_carve(m, B, S, &w);
  int rc = ctx->ensure_ws(m.off);
  if (rc) return rc;
  Arena a(ctx->ws, SIZE_MAX, false);
  ds_carve(a, B, S, &w);
  const int nb = (S + eqk::Q - 1) / eqk::Q;
  rc = eqk::eq_run(ctx, d.f, x, S, S, n_in, nullptr, B, nb, nb, w.e, w.s, nullptr, w.h, S, st);
  if (rc) return rc;
  return cpk::cp_run(ctx, d.p, x, S, S, n_in, nullptr, B, S, S, w.w, y, S, reduction_db, st, cpk::CpSplit{w.h, d.range});
}

}  // namespace

int vtts_deess(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float freq_hz, float threshold_db, float ratio,
               float knee_db, float attack_ms, float release_ms, float range_db, float* y_dev, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  DsParams d;
  const int rc = ds_args(ctx, "deess", B, S, rate, freq_hz, threshold_db, ratio, knee_db, attack_ms, release_ms, range_db, &d);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "deess: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return ds_launch(ctx, d, x_dev, n_dev, B, S, y_dev, reduction_db_dev, (cudaStream_t)stream);
}

int vtts_deess_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float freq_hz, float threshold_db, float ratio,
                    float knee_db, float attack_ms, float release_ms, float range_db, float* y, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  DsParams d;
  int rc = ds_args(ctx, "deess_host", B, S, rate, freq_hz, threshold_db, ratio, knee_db, attack_ms, release_ms, range_db, &d);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("deess_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_r = hs.out((size_t)B * 4, reduction_db), o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return ds_launch(ctx, d, hs.x(), hs.n(), B, S, hs.dev<float>(o_y), hs.dev<float>(o_r), st); });
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and released in E (the same: no lookahead).  The equalizer reads
// the window (its rows, table 0); the detector reads x_dev and h in place (its rows, table 1).
struct vtts_deesser_stream : SampleStream<eqk::EqRow, cpk::CpRow> {
  using SampleStream::SampleStream;
  DsParams d{};
  int ld_k = 0;
  float *e = nullptr, *s = nullptr, *carry = nullptr;   // the equalizer stream's block states and carried state
  float* h = nullptr;                                   // [S][F] the high band of the push's new samples
  cpk::CpBufs w{};
};

int vtts_deesser_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float freq_hz, float threshold_db, float ratio,
                               float knee_db, float attack_ms, float release_ms, float range_db, vtts_deesser_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "deesser_stream_create", out, true, max_streams, max_chunk_samples);
  if (rc) return rc;
  DsParams d;
  rc = ds_params(ctx, "deesser_stream_create", rate, freq_hz, threshold_db, ratio, knee_db, attack_ms, release_ms, range_db, &d);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_deesser_stream> ds(new vtts_deesser_stream(ctx, max_streams, max_chunk_samples, eqk::Q));
  ds->d = d;
  ds->ld_k = eqk::eq_stream_blocks(max_chunk_samples);
  const size_t S = max_streams;
  rc = stream_alloc(ctx, "deesser_stream_create", *ds, [&](Arena& a) {
    ds->carve_window(a);
    ds->e = a.take<float>(S * ds->ld_k * eqk::NS);
    ds->s = a.take<float>(S * ds->ld_k * eqk::NS);
    ds->carry = a.take<float>(S * eqk::NS);
    ds->h = a.take<float>(S * max_chunk_samples);
    cpk::cp_carve(a, S, cpk::cp_blocks_max(max_chunk_samples), &ds->w);
    ds->w.carry_r = a.take<float4>(S);
    ds->w.carry_a = a.take<float4>(S);
    ds->w.carry_y1 = a.take<float>(S);
    ds->w.carry_yl = a.take<float>(S);
    ds->w.carry_max = a.take<float>(S);
    ds->carve_tables(a);
  });
  if (rc) return rc;
  *out = ds.release();
  return VTTS_OK;
}

int vtts_deesser_stream_destroy(vtts_ctx* ctx, vtts_deesser_stream* ds) { return stream_destroy(ctx, "deesser_stream_destroy", ds); }

int vtts_deesser_stream_push(vtts_ctx* ctx, vtts_deesser_stream* ds, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                             float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "deesser_stream_push", ds, x_dev && n_new && flags && y_dev && n_out && reduction_db_dev);
  if (rc) return rc;
  const SlotState& sl = ds->slots;
  rc = sl.check(ctx, "deesser_stream_push", ds->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = ds->S;

  // ---- host bookkeeping: every sample is released in the push that brings it ----
  eqk::EqRow* erows = ds->rows<0>();
  cpk::CpRow* crows = ds->rows<1>();
  std::vector<long long> E1(S);
  long long max_k = 0, max_rn = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    erows[s] = eqk::eq_stream_row(P0, P1, begin);
    crows[s] = cpk::cp_stream_row(P0, P1, begin);
    E1[s] = P1;
    n_out[s] = (int32_t)(P1 - P0);
    max_k = std::max(max_k, (long long)erows[s].nk);
    max_rn = std::max(max_rn, crows[s].rn);
  }
  if (max_k > ds->ld_k) return ctx->fail(VTTS_ERR_CUDA, "deesser_stream_push: %lld blocks (internal bound %d)", max_k, ds->ld_k);

  // ---- device: one table copy, the window step, the equalizer's three launches into h, the compressor's six ----
  rc = ds->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  rc = eqk::eq_run(ctx, ds->d.f, ds->win, ds->cap, ds->cap, nullptr, ds->d_rows<0>(), S, max_k, ds->ld_k, ds->e, ds->s, ds->carry, ds->h,
                   ds->F, st);
  if (rc) return rc;
  rc = cpk::cp_run(ctx, ds->d.p, x_dev, ds->F, ds->F, nullptr, ds->d_rows<1>(), S, max_rn, max_rn, ds->w, y_dev, ds->F, reduction_db_dev, st,
                   cpk::CpSplit{ds->h, ds->d.range});
  if (rc) return rc;
  ds->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_deesser_stream_push_host(vtts_ctx* ctx, vtts_deesser_stream* ds, const float* x, const int32_t* n_new, const uint8_t* flags,
                                  float* y, int32_t* n_out, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "deesser_stream_push_host", ds, x && y && reduction_db);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)ds->S * ds->F * 4), o_y = hs.out((size_t)ds->S * ds->F * 4, y), o_r = hs.out((size_t)ds->S * 4, reduction_db);
  return hs.run([&](cudaStream_t st) {
    return vtts_deesser_stream_push(ctx, ds, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, hs.dev<float>(o_r), st);
  });
}
