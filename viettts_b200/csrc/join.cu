// Joined utterances: texts of several sentences, each sentence a token row planned and run through the acoustic model
// on its own, the emitted frames of a text's sentences gathered into one mel row and vocoded once (vtts_tts_joined_host).
#include <climits>

#include "stream_common.cuh"

namespace {
constexpr int Q = vc::MEL / 4;   // float4 per mel frame

// the key of the acoustic launch of rows [128c, 128c + 128) in SEED mode (engine.py _chunk_seed)
uint64_t chunk_seed(uint64_t seed, int chunk) { return seed ^ ((uint64_t)chunk * 0x9E3779B97F4A7C15ull); }

// out [G][n_max][80]: frame t of text g is frame t - start[s] of sentence s, the last sentence of the text that starts at
// or before t (a zero-frame sentence shares its start with the next one, so it is never picked), read at frame
// src[s] + t - start[s] of the acoustic mel; frames at or past n_frames[g] are zero.
// tbl: int32 start [B] | src [B] | group_start [G + 1] | n_frames [G]
__global__ void __launch_bounds__(256) join_kernel(const float4* __restrict__ mel, const int32_t* __restrict__ tbl, int B, int G,
                                                   int n_max, float4* __restrict__ out) {
  const int32_t* start = tbl;
  const int32_t* src = tbl + B;
  const int32_t* gs = tbl + 2 * B;
  const int32_t* nf = gs + G + 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_max * Q) return;
  const int t = i / Q, q = i - t * Q;
  for (int g = blockIdx.y; g < G; g += gridDim.y) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < nf[g]) {
      int lo = gs[g], hi = gs[g + 1] - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (start[mid] <= t) lo = mid;
        else hi = mid - 1;
      }
      v = mel[((size_t)src[lo] + (t - start[lo])) * Q + q];
    }
    out[((size_t)g * n_max + t) * Q + q] = v;
  }
}
}  // namespace

extern "C" int vtts_tts_joined_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, const int32_t* group_start,
                                    int G, float silence_duration, int dropout_mode, uint64_t seed, int max_frames, float* dur_sec_out,
                                    int32_t* sent_start_out, int32_t* n_frames_out, int32_t* n_max_out, float* wav) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens || !group_start || !sent_start_out || !n_frames_out || !n_max_out || !wav || B < 1 || L < 1 || G < 1 || max_frames < 1)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: bad argument");
  if (dropout_mode != VTTS_DROPOUT_OFF && dropout_mode != VTTS_DROPOUT_SEED && dropout_mode != VTTS_DROPOUT_REFERENCE)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: dropout_mode must be OFF, SEED or REFERENCE (the frame count is not known to the caller)");
  if (L > vtts_acoustic_max_tokens())
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: L=%d tokens per sentence, the acoustic model takes at most %d", L,
                     vtts_acoustic_max_tokens());
  if (group_start[0] != 0 || group_start[G] != B)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: group_start must run from 0 to B=%d, got %d .. %d", B, group_start[0], group_start[G]);
  for (int g = 0; g < G; ++g)
    if (group_start[g + 1] <= group_start[g])
      return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: group_start is not strictly increasing at %d (%d, %d)", g, group_start[g],
                       group_start[g + 1]);
  std::vector<float> frames((size_t)B * L);
  std::vector<int32_t> nf_ac(B), ne(B);
  int rc = vtts_tts_plan(ctx, tokens, lengths, B, L, silence_duration, dur_sec_out, frames.data(), nf_ac.data(), ne.data());
  if (rc) return rc;

  // each sentence's first frame in its text; a text's frame count is the sum of its sentences' emitted frames
  long long n_max = 0;
  for (int g = 0; g < G; ++g) {
    long long t = 0;
    for (int b = group_start[g]; b < group_start[g + 1]; ++b) {
      sent_start_out[b] = (int32_t)std::min<long long>(t, INT_MAX);
      t += ne[b];
    }
    n_frames_out[g] = (int32_t)std::min<long long>(t, INT_MAX);
    n_max = std::max(n_max, t);
  }
  *n_max_out = (int32_t)std::min<long long>(n_max, INT_MAX);
  if (n_max < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: the sentences' frames sum to less than one frame");
  if (n_max > max_frames)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: needs %lld frames, caller buffer holds %d (n_max_out is set: retry with that size)",
                     n_max, max_frames);
  const int T = (int)n_max;

  // acoustic launches of at most 128 rows, each as wide as its longest row; a launch none of whose rows emits is skipped
  const int C = (B + vc::LAUNCH_ROWS - 1) / vc::LAUNCH_ROWS;
  std::vector<int> Nc(C, 0);
  std::vector<long long> base(C + 1, 0);
  std::vector<int32_t> tbl((size_t)2 * B + 2 * G + 1);
  for (int c = 0; c < C; ++c) {
    const int b0 = c * vc::LAUNCH_ROWS, b1 = std::min(B, b0 + vc::LAUNCH_ROWS);
    int n = 0, emit = 0;
    for (int b = b0; b < b1; ++b) {
      n = std::max(n, nf_ac[b]);
      emit = std::max(emit, ne[b]);
    }
    Nc[c] = emit > 0 ? n : 0;
    for (int b = b0; b < b1; ++b) tbl[B + b] = (int32_t)(base[c] + (long long)(b - b0) * Nc[c]);
    base[c + 1] = base[c] + (long long)(b1 - b0) * Nc[c];
  }
  if (base[C] > INT_MAX) return ctx->fail(VTTS_ERR_BAD_ARG, "tts_joined_host: %lld acoustic frames in one call", base[C]);
  memcpy(tbl.data(), sent_start_out, (size_t)B * 4);
  memcpy(tbl.data() + 2 * B, group_start, (size_t)(G + 1) * 4);
  memcpy(tbl.data() + 2 * B + G + 1, n_frames_out, (size_t)G * 4);

  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t wav_b = (size_t)G * T * vc::HOP * 4;
  HostStage hs(ctx);
  const size_t o_tok = hs.in(tokens, (size_t)B * L * 4), o_len = hs.in(lengths, lengths ? (size_t)B * 4 : 0);
  const size_t o_dur = hs.in(frames.data(), frames.size() * 4), o_nf = hs.in(nf_ac.data(), (size_t)B * 4);
  const size_t o_tbl = hs.in(tbl.data(), tbl.size() * 4);
  const size_t o_wav = hs.out(wav_b);
  const size_t o_mel = hs.scratch((size_t)base[C] * vc::MEL * 4), o_join = hs.scratch((size_t)G * T * vc::MEL * 4);
  rc = hs.upload();
  if (rc) return rc;
  float* mel = hs.dev<float>(o_mel);
  for (int c = 0; c < C && !rc; ++c) {
    if (Nc[c] < 1) continue;
    const size_t b0 = (size_t)c * vc::LAUNCH_ROWS;
    const int nb = std::min(B - (int)b0, vc::LAUNCH_ROWS);
    rc = vtts_acoustic_forward(ctx, hs.dev<const int32_t>(o_tok) + b0 * L, lengths ? hs.dev<const int32_t>(o_len) + b0 : nullptr,
                               hs.dev<const float>(o_dur) + b0 * L, hs.dev<const int32_t>(o_nf) + b0, nullptr, dropout_mode,
                               dropout_mode == VTTS_DROPOUT_SEED ? chunk_seed(seed, c) : seed, nb, L, Nc[c],
                               mel + (size_t)base[c] * vc::MEL, hs.st);
  }
  if (rc) return rc;
  const int32_t* d_tbl = hs.dev<const int32_t>(o_tbl);
  dim3 grid((T * Q + 255) / 256, std::min(G, 65535));
  join_kernel<<<grid, 256, 0, hs.st>>>(reinterpret_cast<const float4*>(mel), d_tbl, B, G, T, hs.dev<float4>(o_join));
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  // the generator workspace replaces the acoustic one: growing it frees memory the acoustic launches may still use
  if (vtts_hifigan_ws_bytes(G, T) > ctx->ws_bytes) VTTS_CUDA(cudaStreamSynchronize(hs.st));
  rc = vtts_hifigan_forward(ctx, hs.dev<const float>(o_join), d_tbl + 2 * B + G + 1, G, T, hs.dev<float>(o_wav), hs.st);
  if (!rc) rc = hs.fetch(o_wav, wav, wav_b);
  return rc ? rc : hs.finish();
}
