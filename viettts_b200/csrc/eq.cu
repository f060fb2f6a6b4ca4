// Equalizer: a cascade of K <= 8 second-order sections over one mono row, fp32 on the device in every vtts_precision
// mode (oracle/eq_oracle.py states it in float64):
//   y = scipy.signal.sosfilt(sos, x) from zero state at sample 0, sos [K][6] = b0 b1 b2 a0 a1 a2;  outputs past n are 0.
//
// Section form.  Every section runs as the trapezoidal (TPT) state-variable filter of its own bilinear transform
// (Simper's linear SVF, the form of the loudness meter's high-pass): with the coefficients normalized by a0,
//   g^2 = (1 + a1 + a2) / (1 - a1 + a2),  k = 2 g (1 - a2) / (1 + a1 + a2)   (both exist for every stable section),
//   n2 = g^2 (b0 - b1 + b2) / c0,  n1 = 2 g (b0 - b2) / c0,  n0 = (b0 + b1 + b2) / c0,  c0 = 1 + a1 + a2,
//   m0 = n2,  m1 = n1 - m0 k,  m2 = n0 - m0,
// derived in double and rounded to fp32 once.  Per sample, state (s1, s2): v3 = x - s2, v1 = d s1 + g d v3,
// v2 = s2 + g d s1 + g^2 d v3 (d = 1 / (1 + g (g + k))), s1 = 2 v1 - s1, s2 = 2 v2 - s2, y = m0 x + m1 v1 + m2 v2.
// Rounded to fp32, direct-form coefficients of a low-frequency section move its poles (a1 = -2 + O(g), a2 = 1 - O(g));
// the state-variable coefficients keep them to fp32 precision.
//
// Invariant (as in loudness.cu and limiter.cu).  Blocks of Q = 1024 samples fixed by absolute sample index.  The
// cascade state entering block k is s_k, s_k+1 = M s_k + e_k, with e_k the block's end state from zero (a fixed fp32
// function of its samples) and M = A^Q (A the 2K x 2K block-lower-triangular one-sample transition of the cascade,
// powered in double and rounded to fp32).  Every output of block k is a fixed fp32 function of s_k and the block's
// samples, so a row gives the same bits alone, in any batch position, in every precision mode and through the stream.
//
// Block kernel.  One warp per (row, block), lane l holding samples [32 l, 32 l + 32) in registers (staged through shared
// memory so the global loads and stores coalesce).  For each section in turn: every lane filters its segment from zero,
// a five-step Hillis-Steele scan with the section's 2 x 2 transitions A_j^(32 2^d) composes the lane end states into
// each lane's entering state (lane 0 enters with zero, or with s_k in the output pass), and every lane re-filters its
// segment from it, which gives the section's exact outputs as the next section's input.  Samples past the row's end
// read as 0; only later samples depend on them, so no lane needs a bound.  The kernel runs twice: from zero (the lane
// holding a complete block's last sample writes e_k) and from s_k (y).
//
// Chain kernel.  One warp per row: the lanes stage 32 blocks' e_k in shared memory, then walk s_k+1 = M s_k + e_k over
// them with lane a < 2K holding state row a and row a of M (the 2K states reach every lane by shuffles), and store the
// 32 entering states.
//
// Stream.  Per slot a window of Q carried samples plus one chunk (the resample stream's window step) and the cascade
// state at the last complete block boundary.  A push re-runs the slot's incomplete block from that boundary and writes
// the outputs of every sample it brought: an IIR filter needs no lookahead.  Every push issues the same four launches.
#include "eq_kernels.cuh"

using namespace eqk;

namespace {

// ---- the designer ---------------------------------------------------------------------------------------------------

void put(double* row, double b0, double b1, double b2, double a0, double a1, double a2) {
  const double v[6] = {b0 / a0, b1 / a0, b2 / a0, 1.0, a1 / a0, a2 / a0};
  std::memcpy(row, v, sizeof(v));
}

}  // namespace

int vtts_eq_design(int kind, int rate, double f0, double q, double gain_db, int order, double* sos, int* n_sections) {
  if (!sos || !n_sections) return VTTS_ERR_BAD_ARG;
  if (rate < 8000 || rate > 192000 || !(f0 >= 10.0 && f0 <= 0.45 * rate)) return VTTS_ERR_BAD_ARG;
  const double pi = 3.14159265358979323846;
  const double w0 = 2.0 * pi * f0 / rate, cw = std::cos(w0), sw = std::sin(w0);
  const bool gain_ok = gain_db >= -24.0 && gain_db <= 24.0, q_ok = q >= 0.1 && q <= 30.0;
  const double A = std::pow(10.0, gain_db / 40.0);
  switch (kind) {
    case VTTS_EQ_HIGHPASS:
    case VTTS_EQ_LOWPASS: {
      // Butterworth: pairs s^2 + 2 sin(pi (2i + 1) / 2N) s + 1 and, for odd N, s + 1, through the bilinear transform
      // prewarped to f0 (s = (z - 1) / (K (z + 1)), K = tan(pi f0 / rate))
      if (order < 1 || order > 8) return VTTS_ERR_BAD_ARG;
      const bool hp = kind == VTTS_EQ_HIGHPASS;
      const double K = std::tan(pi * f0 / rate), K2 = K * K;
      int j = 0;
      for (int i = 0; i < order / 2; ++i, ++j) {
        const double z2 = 2.0 * std::sin(pi * (2 * i + 1) / (2.0 * order));
        const double a0 = 1.0 + z2 * K + K2, a1 = 2.0 * (K2 - 1.0), a2 = 1.0 - z2 * K + K2;
        if (hp)
          put(sos + 6 * j, 1.0, -2.0, 1.0, a0, a1, a2);
        else
          put(sos + 6 * j, K2, 2.0 * K2, K2, a0, a1, a2);
      }
      if (order % 2) {
        if (hp)
          put(sos + 6 * j, 1.0, -1.0, 0.0, 1.0 + K, K - 1.0, 0.0);
        else
          put(sos + 6 * j, K, K, 0.0, 1.0 + K, K - 1.0, 0.0);
        ++j;
      }
      *n_sections = j;
      return VTTS_OK;
    }
    case VTTS_EQ_LOWSHELF:
    case VTTS_EQ_HIGHSHELF: {
      // RBJ Audio EQ Cookbook shelves, q = the shelf slope S in (0, 1]
      if (!(q > 0.0 && q <= 1.0) || !gain_ok) return VTTS_ERR_BAD_ARG;
      const double alpha = sw / 2.0 * std::sqrt((A + 1.0 / A) * (1.0 / q - 1.0) + 2.0), ra = 2.0 * std::sqrt(A) * alpha;
      if (kind == VTTS_EQ_LOWSHELF)
        put(sos, A * ((A + 1) - (A - 1) * cw + ra), 2 * A * ((A - 1) - (A + 1) * cw), A * ((A + 1) - (A - 1) * cw - ra),
            (A + 1) + (A - 1) * cw + ra, -2 * ((A - 1) + (A + 1) * cw), (A + 1) + (A - 1) * cw - ra);
      else
        put(sos, A * ((A + 1) + (A - 1) * cw + ra), -2 * A * ((A - 1) + (A + 1) * cw), A * ((A + 1) + (A - 1) * cw - ra),
            (A + 1) - (A - 1) * cw + ra, 2 * ((A - 1) - (A + 1) * cw), (A + 1) - (A - 1) * cw - ra);
      *n_sections = 1;
      return VTTS_OK;
    }
    case VTTS_EQ_PEAKING: {
      if (!q_ok || !gain_ok) return VTTS_ERR_BAD_ARG;
      const double alpha = sw / (2.0 * q);
      put(sos, 1.0 + alpha * A, -2.0 * cw, 1.0 - alpha * A, 1.0 + alpha / A, -2.0 * cw, 1.0 - alpha / A);
      *n_sections = 1;
      return VTTS_OK;
    }
    case VTTS_EQ_NOTCH: {
      if (!q_ok) return VTTS_ERR_BAD_ARG;
      const double alpha = sw / (2.0 * q);
      put(sos, 1.0, -2.0 * cw, 1.0, 1.0 + alpha, -2.0 * cw, 1.0 - alpha);
      *n_sections = 1;
      return VTTS_OK;
    }
    default:
      return VTTS_ERR_BAD_ARG;
  }
}

namespace {

// the batch shape and filter of a one-shot call of entry point `who`
int eq_args(vtts_ctx* ctx, const char* who, int B, int S, const double* sos, int K, EqFilter* f) {
  const int rc = batch_check(ctx, who, B, S, S_MAX);
  return rc ? rc : eq_filter(ctx, who, sos, K, f);
}

int eq_launch(vtts_ctx* ctx, const EqFilter& f, const float* x, const int32_t* n_in, int B, int S, float* y, cudaStream_t st) {
  const int nb = (S + Q - 1) / Q;
  const size_t es_b = al((size_t)B * nb * NS * 4);
  const int rc = ctx->ensure_ws(2 * es_b);
  if (rc) return rc;
  float* e = (float*)ctx->ws;
  float* s = (float*)((char*)ctx->ws + es_b);
  return eq_run(ctx, f, x, S, S, n_in, nullptr, B, nb, nb, e, s, nullptr, y, S, st);
}

}  // namespace

int vtts_eq(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const double* sos, int K, float* y_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  EqFilter f;
  const int rc = eq_args(ctx, "eq", B, S, sos, K, &f);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "eq: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return eq_launch(ctx, f, x_dev, n_dev, B, S, y_dev, (cudaStream_t)stream);
}

int vtts_eq_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const double* sos, int K, float* y) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  EqFilter f;
  int rc = eq_args(ctx, "eq_host", B, S, sos, K, &f);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("eq_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_y = hs.out((size_t)B * S * 4, y);
  return hs.run([&](cudaStream_t st) { return eq_launch(ctx, f, hs.x(), hs.n(), B, S, hs.dev<float>(o_y), st); });
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and released in E (the same: no lookahead).
struct vtts_eq_stream : SampleStream<EqRow> {
  using SampleStream::SampleStream;
  EqFilter f{};
  int ld_k = 0;
  float *e = nullptr, *s = nullptr, *carry = nullptr;
};

int vtts_eq_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, const double* sos, int K, vtts_eq_stream** out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "eq_stream_create", out, true, max_streams, max_chunk_samples);
  if (rc) return rc;
  EqFilter f;
  rc = eq_filter(ctx, "eq_stream_create", sos, K, &f);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_eq_stream> es(new vtts_eq_stream(ctx, max_streams, max_chunk_samples, Q));
  es->f = f;
  es->ld_k = eq_stream_blocks(max_chunk_samples);
  const size_t S = max_streams;
  rc = stream_alloc(ctx, "eq_stream_create", *es, [&](Arena& a) {
    es->carve_window(a);
    es->e = a.take<float>(S * es->ld_k * NS);
    es->s = a.take<float>(S * es->ld_k * NS);
    es->carry = a.take<float>(S * NS);
    es->carve_tables(a);
  });
  if (rc) return rc;
  *out = es.release();
  return VTTS_OK;
}

int vtts_eq_stream_destroy(vtts_ctx* ctx, vtts_eq_stream* es) { return stream_destroy(ctx, "eq_stream_destroy", es); }

int vtts_eq_stream_push(vtts_ctx* ctx, vtts_eq_stream* es, const float* x_dev, const int32_t* n_new, const uint8_t* flags, float* y_dev,
                        int32_t* n_out, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "eq_stream_push", es, x_dev && n_new && flags && y_dev && n_out);
  if (rc) return rc;
  const SlotState& sl = es->slots;
  rc = sl.check(ctx, "eq_stream_push", es->F, n_new, flags);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = es->S;

  // ---- host bookkeeping: every sample is released in the push that brings it ----
  EqRow* rows = es->rows<0>();
  std::vector<long long> E1(S);
  long long max_k = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1;
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    const EqRow r = eq_stream_row(P0, P1, begin);
    rows[s] = r;
    E1[s] = P1;
    n_out[s] = (int32_t)(P1 - P0);
    max_k = std::max(max_k, (long long)r.nk);
  }
  if (max_k > es->ld_k) return ctx->fail(VTTS_ERR_CUDA, "eq_stream_push: %lld blocks (internal bound %d)", max_k, es->ld_k);

  // ---- device: one table copy, window step, the three filter launches (four in all) ----
  rc = es->upload(n_new, flags, x_dev, st);
  if (rc) return rc;
  rc = eq_run(ctx, es->f, es->win, es->cap, es->cap, nullptr, es->d_rows<0>(), S, max_k, es->ld_k, es->e, es->s, es->carry, y_dev, es->F, st);
  if (rc) return rc;
  es->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_eq_stream_push_host(vtts_ctx* ctx, vtts_eq_stream* es, const float* x, const int32_t* n_new, const uint8_t* flags, float* y,
                             int32_t* n_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  const int rc = stream_args(ctx, "eq_stream_push_host", es, x && y);
  if (rc) return rc;
  const size_t b = (size_t)es->S * es->F * 4;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, b), o_y = hs.out(b, y);
  return hs.run([&](cudaStream_t st) { return vtts_eq_stream_push(ctx, es, hs.dev<const float>(o_x), n_new, flags, hs.dev<float>(o_y), n_out, st); });
}
