// Background bed under a mono speech row, ducked by the voice, fp32 on the device in every vtts_precision mode
// (oracle/bed_oracle.py states it in float64):
//   y_L = the compressor's detector (ratio 20, knee 6 dB, threshold T, attack, release) on L = 20 log10 |x|, x = 0 from
//   the row's end n on;  y^_L = min(y_L, D);  g = 10^(-y^_L / 20);
//   bl[t] = b[u], u = (t + o) mod P, P = Nb - C, crossfaded over u < C as sin(pi u / 2C) b[u] + cos(pi u / 2C) b[P + u];
//   e[t] = the raised-cosine fade-in over [0, Fi) times the raised-cosine fade-out over the tail [n, n + Tt);
//   y[t] = x[t] + g e bl for t < n + Tt;  reduction = -max y^_L.  A row without a bed (index -1) is x, without a tail.
//
// Composition.  One gather writes the key row, x with zeros from n on, [rows][width]; the detector is the compressor's
// six launches (compressor_kernels.cuh) over that row, with the apply rule CpDuck: the cap min(y_L, D), and y =
// fmaf(g e, bl, x) from the bed bank at the absolute sample index, x itself for rows without a bed.  The compressor's
// block invariant holds unchanged (256-sample blocks fixed by absolute index) and the bed, the crossfade and both
// envelopes are functions of the absolute index alone, so a row gives the same bits alone, in any batch position, in
// every precision mode and through the stream at any push pattern.
//
// Stream.  No lookahead: every push releases the samples it brings, and the push with END also releases the row's Tt
// tail samples (the key is zero there, so the detector releases and the bed swells back under the fade-out).  Per slot
// the compressor stream's state and the bed index read with BEGIN.  Every push issues one table copy, the gather and
// the compressor's six launches.
#include <climits>

#include "compressor_kernels.cuh"

namespace {

constexpr int BD_MAX_BEDS = 8;
constexpr float BD_RATIO = 20.f, BD_KNEE = 6.f;
constexpr int GATHER_THREADS = 256;

// per row: where its bed lies in the bank and where its voice ends
struct BdRow {
  long long xend;    // absolute index of the tail's first sample (LLONG_MAX while a stream row is open)
  long long off;     // bank offset of the row's bed
  int nx;            // key samples of the call taken from x (the rest are 0)
  int bed;           // bank entry, -1 for none
  int len;           // Nb of the row's bed
  int kn;            // key samples of the call: nx, and the tail with END
};
static_assert(sizeof(BdRow) % 16 == 0, "table entries keep 16-byte alignment");

struct BdParams {
  cpk::CpParams p;   // the detector (ratio 20, knee 6 dB, makeup 1)
  float D;           // the duck depth, dB
  int Fi, Tt, C;     // fade-in, tail and crossfade, samples
  long long o;       // start offset into the loop, samples
};

// the apply rule of the ducker: the key is x (0 past the voice), y = x + g e bl
struct CpDuck {
  const BdRow* rows;
  const float* bank;
  float D;
  int Fi, Tt, C;
  long long o;
  __host__ __device__ const float* source(const float* x) const { return x; }
  __device__ __forceinline__ float level(const float*, long long, float v) const { return v; }
  __device__ __forceinline__ float cap(int b, float yl) const { return rows[b].bed < 0 ? 0.f : fminf(yl, D); }
  __device__ __forceinline__ float out(const cpk::CpParams&, int b, long long t, float v, float, float, float g) const {
    const BdRow r = rows[b];
    if (r.bed < 0) return v;
    float e = 1.f;
    if (t < Fi) e = 0.5f - 0.5f * cospif((float)t / (float)Fi);
    if (t >= r.xend) e *= 0.5f + 0.5f * cospif((float)(t - r.xend + 1) / (float)Tt);
    const long long P = r.len - C;
    const int u = (int)((t + o) % P);
    const float* bb = bank + r.off;
    float bl = bb[u];
    if (u < C) {
      const float w = (float)u / (float)(2 * C);
      bl = fmaf(sinpif(w), bl, cospif(w) * bb[P + u]);
    }
    return fmaf(g * e, bl, v);
  }
};

// key[row][t] = x[row][t] for t < nx, else 0, over the kn samples the detector reads.  One-shot rows (n2 != null) take
// nx from n_in (clamped to [0, S]; null: S), complete their table entry and write the detector's length n2 = kn = nx
// (+ Tt with a bed).
__global__ void __launch_bounds__(GATHER_THREADS) bd_key_kernel(const float* __restrict__ x, long long x_ld, int S,
                                                                const int* __restrict__ n_in, int Tt, BdRow* rows, int* n2,
                                                                float* __restrict__ key, int width) {
  const int b = blockIdx.y;
  int nx, kn;
  if (n2) {
    nx = n_in ? min(max(n_in[b], 0), S) : S;
    kn = nx + (rows[b].bed >= 0 ? Tt : 0);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      rows[b].xend = nx;
      rows[b].nx = nx;
      rows[b].kn = kn;
      n2[b] = kn;
    }
  } else {
    nx = rows[b].nx;
    kn = rows[b].kn;
  }
  const float* xr = x + (size_t)b * x_ld;
  float* kr = key + (size_t)b * width;
  for (int t = blockIdx.x * GATHER_THREADS + threadIdx.x; t < kn; t += gridDim.x * GATHER_THREADS) kr[t] = t < nx ? xr[t] : 0.f;
}

int bd_gather(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, int Tt, BdRow* rows, int* n2, float* key, int width,
              int B, cudaStream_t st) {
  const dim3 grid((unsigned)std::min((width + GATHER_THREADS - 1) / GATHER_THREADS, 64), B);
  bd_key_kernel<<<grid, GATHER_THREADS, 0, st>>>(x, x_ld, S, n_in, Tt, rows, n2, key, width);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// every bad argument fails here, before anything is launched
int bd_params(vtts_ctx* ctx, const char* who, int rate, const float* bank_dev, const long long* offsets, const int32_t* lengths, int K,
              float duck_db, float threshold_db, float attack_ms, float release_ms, int fade_in, int tail, int xfade, long long offset,
              BdParams* d) {
  int rc = cpk::cp_params(ctx, who, rate, threshold_db, BD_RATIO, BD_KNEE, attack_ms, release_ms, 0.f, &d->p);
  if (rc) return rc;
  if (!(duck_db >= 0.f && duck_db <= 40.f)) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: duck %g dB (in [0, 40])", who, (double)duck_db);
  if (fade_in < 0 || fade_in > 5 * rate) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: fade_in %d samples (in [0, 5 rate])", who, fade_in);
  if (tail < 0 || tail > 10 * rate) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: tail %d samples (in [0, 10 rate])", who, tail);
  if (xfade < 0 || xfade > rate) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: xfade %d samples (in [0, rate])", who, xfade);
  if (K < 1 || K > BD_MAX_BEDS) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: %d beds (1..%d)", who, K, BD_MAX_BEDS);
  if (!bank_dev || !offsets || !lengths) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null bank pointer", who);
  for (int k = 0; k < K; ++k) {
    const long long n = lengths[k];
    if (n < rate / 2 || n > 600LL * rate || offsets[k] < 0)
      return ctx->fail(VTTS_ERR_BAD_ARG, "%s: bed %d: %lld samples at %lld (0.5 s to 600 s at rate %d)", who, k, n, offsets[k], rate);
    if (2LL * xfade >= n) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: bed %d: 2 xfade = %d must be below its %lld samples", who, k, 2 * xfade, n);
    if (offset < 0 || offset >= n)
      return ctx->fail(VTTS_ERR_BAD_ARG, "%s: offset %lld samples outside bed %d's [0, %lld)", who, offset, k, n);
  }
  d->D = duck_db;
  d->Fi = fade_in;
  d->Tt = tail;
  d->C = xfade;
  d->o = offset;
  return VTTS_OK;
}

CpDuck bd_rule(const BdParams& d, const BdRow* rows, const float* bank) { return CpDuck{rows, bank, d.D, d.Fi, d.Tt, d.C, d.o}; }

BdRow bd_row(int bed, const long long* offsets, const int32_t* lengths) {
  BdRow r{};
  r.bed = bed;
  r.off = bed >= 0 ? offsets[bed] : 0;
  r.len = bed >= 0 ? lengths[bed] : 0;
  return r;
}

int bd_bed_check(vtts_ctx* ctx, const char* who, const int32_t* bed, int B, int K) {
  if (!bed) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null bed index array", who);
  for (int b = 0; b < B; ++b)
    if (bed[b] < -1 || bed[b] >= K) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: bed[%d]=%d outside [-1, %d]", who, b, bed[b], K - 1);
  return VTTS_OK;
}

// the one-shot workspace: the row table, the detector lengths, the key rows, the compressor's buffers
struct BdBufs {
  BdRow* rows;
  int* n2;
  float* key;
  cpk::CpBufs w;
};

void bd_carve(Arena& a, int B, int W, BdBufs* d) {
  d->rows = a.take<BdRow>(B);
  d->n2 = a.take<int>(B);
  d->key = a.take<float>((size_t)B * W);
  d->w = cpk::CpBufs{};
  cpk::cp_carve(a, B, cpk::cp_blocks_max(W), &d->w);
}

// the parameters, batch shape and bed indices of a one-shot call of entry point `who`
int bd_args(vtts_ctx* ctx, const char* who, int B, int S, int rate, const float* bank_dev, const long long* offsets, const int32_t* lengths,
            int K, const int32_t* bed, float duck_db, float threshold_db, float attack_ms, float release_ms, int fade_in, int tail, int xfade,
            long long offset, BdParams* d) {
  int rc = bd_params(ctx, who, rate, bank_dev, offsets, lengths, K, duck_db, threshold_db, attack_ms, release_ms, fade_in, tail, xfade, offset, d);
  if (!rc) rc = batch_check(ctx, who, B, S, cpk::S_MAX);
  if (!rc && (long long)S + tail > cpk::S_MAX) rc = ctx->fail(VTTS_ERR_BAD_ARG, "%s: S + tail = %lld (at most 2^30)", who, (long long)S + tail);
  return rc ? rc : bd_bed_check(ctx, who, bed, B, K);
}

int bd_launch(vtts_ctx* ctx, const BdParams& d, const float* x, const int32_t* n_in, int B, int S, const float* bank_dev, const long long* offsets,
              const int32_t* lengths, const int32_t* bed, float* y, float* reduction_db, cudaStream_t st) {
  const int W = S + d.Tt;
  Arena m(nullptr, 0, true);
  BdBufs w;
  bd_carve(m, B, W, &w);
  int rc = ctx->ensure_ws(m.off);
  if (rc) return rc;
  Arena a(ctx->ws, SIZE_MAX, false);
  bd_carve(a, B, W, &w);
  std::vector<BdRow> rows(B);
  for (int b = 0; b < B; ++b) rows[b] = bd_row(bed[b], offsets, lengths);
  VTTS_CUDA(cudaMemcpyAsync(w.rows, rows.data(), (size_t)B * sizeof(BdRow), cudaMemcpyHostToDevice, st));
  rc = bd_gather(ctx, x, S, S, n_in, d.Tt, w.rows, w.n2, w.key, W, B, st);
  if (rc) return rc;
  return cpk::cp_run(ctx, d.p, w.key, W, W, w.n2, nullptr, B, W, W, w.w, y, W, reduction_db, st, bd_rule(d, w.rows, bank_dev));
}

}  // namespace

int vtts_bed_mix(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, const float* bank_dev,
                 const long long* offsets, const int32_t* lengths, int K, const int32_t* bed, float duck_db, float threshold_db,
                 float attack_ms, float release_ms, int fade_in, int tail, int xfade, long long offset, float* y_dev,
                 float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  BdParams d;
  const int rc = bd_args(ctx, "bed_mix", B, S, rate, bank_dev, offsets, lengths, K, bed, duck_db, threshold_db, attack_ms, release_ms, fade_in,
                         tail, xfade, offset, &d);
  if (rc) return rc;
  if (!x_dev || !y_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "bed_mix: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  return bd_launch(ctx, d, x_dev, n_dev, B, S, bank_dev, offsets, lengths, bed, y_dev, reduction_db_dev, (cudaStream_t)stream);
}

int vtts_bed_mix_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const float* bank_dev,
                      const long long* offsets, const int32_t* lengths, int K, const int32_t* bed, float duck_db, float threshold_db,
                      float attack_ms, float release_ms, int fade_in, int tail, int xfade, long long offset, float* y, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  BdParams d;
  int rc = bd_args(ctx, "bed_mix_host", B, S, rate, bank_dev, offsets, lengths, K, bed, duck_db, threshold_db, attack_ms, release_ms, fade_in,
                   tail, xfade, offset, &d);
  if (rc) return rc;
  HostStage hs(ctx);
  rc = hs.rows("bed_mix_host", x, n_in, B, S, y != nullptr);
  if (rc) return rc;
  const size_t o_r = hs.out((size_t)B * 4, reduction_db), o_y = hs.out((size_t)B * ((size_t)S + tail) * 4, y);
  return hs.run([&](cudaStream_t st) {
    return bd_launch(ctx, d, hs.x(), hs.n(), B, S, bank_dev, offsets, lengths, bed, hs.dev<float>(o_y), hs.dev<float>(o_r), st);
  });
}

// ---- stream ---------------------------------------------------------------------------------------------------
// The shared slot state counts samples received in P and released in E (E = P + Tt after an END with a bed).  The
// gather reads x_dev in place (table 1) into the key rows [S][F + Tt]; the detector reads those (table 0).
struct vtts_bed_stream : SampleStream<cpk::CpRow, BdRow> {
  using SampleStream::SampleStream;
  BdParams d{};
  const float* bank = nullptr;                 // the caller's bank, valid until destroy
  std::vector<long long> offsets;
  std::vector<int32_t> lengths;
  std::vector<int> bed;                        // each slot's bank entry since its BEGIN
  float* key = nullptr;                        // [S][F + Tt]
  cpk::CpBufs w{};
};

int vtts_bed_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, const float* bank_dev, const long long* offsets,
                           const int32_t* lengths, int K, float duck_db, float threshold_db, float attack_ms, float release_ms, int fade_in,
                           int tail, int xfade, long long offset, vtts_bed_stream** out, int* out_pitch) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = create_check(ctx, "bed_stream_create", out, out_pitch != nullptr, max_streams, max_chunk_samples);
  if (rc) return rc;
  BdParams d;
  rc = bd_params(ctx, "bed_stream_create", rate, bank_dev, offsets, lengths, K, duck_db, threshold_db, attack_ms, release_ms, fade_in,
                     tail, xfade, offset, &d);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<vtts_bed_stream> bs(new vtts_bed_stream(ctx, max_streams, max_chunk_samples, 0));
  bs->d = d;
  bs->bank = bank_dev;
  bs->offsets.assign(offsets, offsets + K);
  bs->lengths.assign(lengths, lengths + K);
  bs->bed.assign(max_streams, -1);
  const size_t S = max_streams, W = (size_t)max_chunk_samples + tail;
  rc = stream_alloc(ctx, "bed_stream_create", *bs, [&](Arena& a) {
    bs->key = a.take<float>(S * W);
    cpk::cp_carve(a, S, cpk::cp_blocks_max((long long)W), &bs->w);
    bs->w.carry_r = a.take<float4>(S);
    bs->w.carry_a = a.take<float4>(S);
    bs->w.carry_y1 = a.take<float>(S);
    bs->w.carry_yl = a.take<float>(S);
    bs->w.carry_max = a.take<float>(S);
    bs->carve_tables(a);
  });
  if (rc) return rc;
  *out_pitch = (int)W;
  *out = bs.release();
  return VTTS_OK;
}

int vtts_bed_stream_destroy(vtts_ctx* ctx, vtts_bed_stream* bs) { return stream_destroy(ctx, "bed_stream_destroy", bs); }

int vtts_bed_stream_push(vtts_ctx* ctx, vtts_bed_stream* bs, const float* x_dev, const int32_t* n_new, const uint8_t* flags, const int32_t* bed,
                         float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "bed_stream_push", bs, x_dev && n_new && flags && bed && y_dev && n_out && reduction_db_dev);
  if (rc) return rc;
  const SlotState& sl = bs->slots;
  const int K = (int)bs->lengths.size();
  rc = sl.check(ctx, "bed_stream_push", bs->F, n_new, flags, [&](int s) {
    if (flags[s] & 1) {
      if (bed[s] < -1 || bed[s] >= K) return ctx->fail(VTTS_ERR_BAD_ARG, "bed_stream_push: bed[%d]=%d outside [-1, %d]", s, bed[s], K - 1);
    } else if (bed[s] != bs->bed[s]) {
      return ctx->fail(VTTS_ERR_BAD_ARG, "bed_stream_push: bed[%d]=%d changes slot %d's bed %d before END", s, bed[s], s, bs->bed[s]);
    }
    return (int)VTTS_OK;
  });
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = bs->S, W = bs->F + bs->d.Tt;

  // ---- host bookkeeping: every sample is released in the push that brings it, the tail with END ----
  cpk::CpRow* crows = bs->rows<0>();
  BdRow* brows = bs->rows<1>();
  std::vector<long long> E1(S);
  long long max_rn = 0;
  for (int s = 0; s < S; ++s) {
    const bool act = SlotState::active(n_new, flags, s), begin = flags[s] & 1, end = flags[s] & 2;
    const int k = act && begin ? bed[s] : bs->bed[s];
    const long long P0 = begin ? 0 : sl.P[s], P1 = P0 + (act ? n_new[s] : 0);
    const long long tl = act && end && k >= 0 ? bs->d.Tt : 0;
    crows[s] = cpk::cp_stream_row(P0, P1 + tl, begin);
    brows[s] = bd_row(k, bs->offsets.data(), bs->lengths.data());
    brows[s].xend = act && end ? P1 : LLONG_MAX;
    brows[s].nx = (int)(P1 - P0);
    brows[s].kn = (int)(P1 + tl - P0);
    E1[s] = P1 + tl;
    n_out[s] = (int32_t)(P1 + tl - P0);
    max_rn = std::max(max_rn, crows[s].rn);
  }

  // ---- device: one table copy, the gather, the compressor's six launches ----
  rc = bs->upload_rows(st);
  if (rc) return rc;
  BdRow* d_brows = const_cast<BdRow*>(bs->d_rows<1>());
  rc = bd_gather(ctx, x_dev, bs->F, bs->F, nullptr, 0, d_brows, nullptr, bs->key, W, S, st);
  if (rc) return rc;
  rc = cpk::cp_run(ctx, bs->d.p, bs->key, W, W, nullptr, bs->d_rows<0>(), S, max_rn, max_rn, bs->w, y_dev, W, reduction_db_dev, st,
                   bd_rule(bs->d, d_brows, bs->bank));
  if (rc) return rc;
  for (int s = 0; s < S; ++s)
    if (SlotState::active(n_new, flags, s) && (flags[s] & 1)) bs->bed[s] = bed[s];
  bs->slots.commit(n_new, flags, E1.data());
  return VTTS_OK;
}

int vtts_bed_stream_push_host(vtts_ctx* ctx, vtts_bed_stream* bs, const float* x, const int32_t* n_new, const uint8_t* flags, const int32_t* bed,
                              float* y, int32_t* n_out, float* reduction_db) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  int rc = stream_args(ctx, "bed_stream_push_host", bs, x && y && reduction_db);
  if (rc) return rc;
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, (size_t)bs->S * bs->F * 4), o_y = hs.out((size_t)bs->S * ((size_t)bs->F + bs->d.Tt) * 4, y),
               o_r = hs.out((size_t)bs->S * 4, reduction_db);
  return hs.run([&](cudaStream_t st) {
    return vtts_bed_stream_push(ctx, bs, hs.dev<const float>(o_x), n_new, flags, bed, hs.dev<float>(o_y), n_out, hs.dev<float>(o_r), st);
  });
}
