// Internal declarations shared by the translation units of libviettts_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>

#include "../../include/viettts_b200.h"

// ---- model constants (vietTTS/nat/config.py:8-59, assets/hifigan/config.json:2-28) ----------
namespace vc {
constexpr int MEL = 80;
constexpr int HOP = 256;
constexpr int NFFT = 1024;
constexpr int NBINS = 513;
constexpr int ENC_D = 256;        // acoustic_encoder_dim
constexpr int ENC_OUT = 512;      // BiLSTM concat
constexpr int DEC_H = 512;        // acoustic_decoder_dim
constexpr int PRENET = 256;
constexpr int POSTNET = 512;
constexpr int VOCAB = 256;
constexpr int SIL_INDEX = 0;      // nat/config.py:26 special_phonemes.index("sil")
constexpr int WORD_END_INDEX = 3; // nat/config.py:28 special_phonemes.index(" ")
constexpr int HG_C0 = 512;        // upsample_initial_channel
constexpr int HG_NSTAGE = 4;
__host__ __device__ constexpr int hg_rate(int i) { return i < 2 ? 8 : 2; }
__host__ __device__ constexpr int hg_upk(int i) { return i < 2 ? 16 : 4; }
__host__ __device__ constexpr int hg_rbk(int j) { return j == 0 ? 3 : (j == 1 ? 7 : 11); }
__host__ __device__ constexpr int hg_dil(int m) { return m == 0 ? 1 : (m == 1 ? 3 : 5); }
}  // namespace vc

#define VTTS_CUDA(expr)                                                                          \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      return ctx->fail(VTTS_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,               \
                       cudaGetErrorString(_e));                                                  \
    }                                                                                            \
  } while (0)

// ---- generic NWC conv problem description (conv1d.cu) ----------------------------------------
struct ConvProb {
  const float* x0;       // input  [B][rows_in][Cin]
  const float* x1;       // extra inputs for pre_mode 2 (sum of three / 3), else null
  const float* x2;
  const float* w;        // [k][Cin][Cout]
  const float* bias;     // [Cout]
  const float* resid;    // [B][rows_out][Cout] or null, added after the activation
  const float* bn_mean;  // eval BatchNorm (all four or none): y = (y-mean)*inv + off
  const float* bn_inv;   //   inv = scale*rsqrt(var+1e-5) precomputed at load
  const float* bn_off;
  float* out;            // [B][rows_out][Cout]
  int k, dil, in_off;    // input row of tap j for output index tau: tau + j*dil + in_off
  int out_stride, out_off;  // output row = tau*out_stride + out_off (transposed-conv phases)
};

struct ConvLaunch {
  ConvProb p[8];
  int nprob;
  int Cin, Cout;
  int B;
  int T_rows;         // tau range per batch row (== allocated input rows)
  int rows_out;       // allocated output rows per batch row
  const int* len;     // int32 [B] or null
  int len_mul;        // valid tau < len[b]*len_mul (clamped to T_rows)
  int pre_mode;       // 0 none, 1 leaky_relu(pre_slope), 2 (x0+x1+x2)/3 then leaky_relu(pre_slope)
  float pre_slope;
  int post_act;       // 0 none, 1 tanh, 2 relu
};

// ---- tensor-core conv (tc_conv.cu) ----------------------------------------------------------------
struct TcProb {
  const float* x0;
  const float* x1;
  const float* x2;
  const void* wpk;       // packed weights (vtts_tc_pack_weights) in the launch's operand format
  const float* bias;     // [N]
  const float* resid;    // rows_out x out_ld or null
  const float* bn_mean;  // eval BatchNorm (all three or none), applied after the bias
  const float* bn_inv;
  const float* bn_off;
  float* out;
  int k, dil, in_off, out_stride, out_off;
  // multi-phase tiles (TcLaunch::nphase > 1): phase ph of this problem uses weights wpk_ph[ph], reads input rows
  // shifted by in_off_ph[ph] and writes output rows tau*out_stride + out_off_ph[ph]; one converted activation
  // tile feeds all phases (ConvTranspose output phases share their input)
  const void* wpk_ph[4];
  int in_off_ph[4];
  int out_off_ph[4];
  // optional per-batch-row bounds [B][3] (device int32): input rows outside [rb[3b], rb[3b+1]) read as zero, and output
  // row tau*out_stride + out_off is written only below rb[3b+2].  Null: rows [0, valid) of the launch for both
  // (vocoder_stream.cu runs "valid" convs over per-slot windows, whose input and output ranges differ)
  const int* rb;
};

struct TcLaunch {
  TcProb p[8];
  int nprob;
  int Cin, N;            // N = output channels of this launch (32/64/128/256)
  int in_ld, out_ld;     // row strides in floats
  int B, T_rows, rows_out;
  const int* len;
  int len_mul;
  int pre_mode;
  float pre_slope;
  int nphase;            // phases per tile (1, 2 or 4); 0 means 1
  int post_act;          // 0 none, 1 tanh, 2 relu (after BN, before the residual)
  int n_valid;           // real output channels of this N tile (<= N); 0 means N
  int f16;               // operand format: 0 = bf16 hi/lo planes, three products (bf16x3); 1 = one fp16 plane, one product
                         // (the generator's VTTS_PRECISION_FP16; plain epilogue only)
  int tile_rows;              // output rows tau per batch row to tile over; 0 means T_rows
  int tiles_per_row, ntiles;  // filled by the launcher
  int* sched;                 // device int[2]: the run-time tile scheduler's counters (vtts_ctx::d_tc_sched)
  int* err;                   // device int: set before trapping on a barrier timeout
  long long* dbg;             // optional [grid][16] per-role stall counters (vtts_debug_tc_stats)
};

// ---- fused ResBlock pair (tc_pair.cu): out = conv2(lrelu(conv1(lrelu(x)) + b1)) + b2 + x, C = N channels ----
struct TcPairProb {
  const float* x;        // [B][T_rows][N] input and residual
  const void* w1pk;      // packed weights of the dilated conv (vtts_tc_pack_weights), in the launch's operand format
  const void* w2pk;      // ... of the dilation-1 conv
  const float* b1;
  const float* b2;
  float* out;            // [B][T_rows][N], must differ from x
  int k, dil;
};

struct TcPairLaunch {
  TcPairProb p[3];
  int nprob;
  int N;
  int B, T_rows;
  const int* len;
  int len_mul;
  float slope;
  int f16;                     // operand format as in TcLaunch (fp16: the default pair form only)
  int tiles_per_row, ntiles;   // filled by the launcher
  int* sched;
  int* err;
  long long* dbg;
};

// Device weights of one model: the checkpoint tensors, fp32 tensors derived from them at load, and the tensor-core
// packing of its convs (vtts_pack_convs: bf16 hi/lo, and for the generator a second, fp16 copy).
struct ModelWeights {
  float* blob = nullptr;        // checkpoint tensors in canonical order, each 256 B aligned
  std::vector<float*> t;
  float* derived = nullptr;     // derived tensors (BN inverses, repacked weights, ...), same layout rules
  std::vector<float*> d;
  void* wpk = nullptr;          // packed convs
  std::vector<void*> wpk_t;     // every N tile of every packed conv, in the order of the packing table
  std::vector<int> tile0;       // index into wpk_t of the first tile of each entry of the packing table
  bool loaded = false;
  // the tiles of packing-table entry `conv`; the tiles of consecutive entries follow each other
  void* const* tiles(int conv) const { return &wpk_t[tile0[conv]]; }
};

struct vtts_ctx {
  int device = 0;
  int precision = 1;            // 0 = strict fp32 (FMA pipe), 1 = bf16x3 on the tensor cores (wgmma, default),
                                // 2 = fp16 operands in the generator, bf16x3 everywhere else (vtts_precision)
  int* d_err = nullptr;
  // tile scheduler counters of the tensor-core launches: [0] next ticket, [1] CTAs done taking tickets.  Each launch
  // leaves them at zero.  One pair serves every launch of the context because a context's tensor-core launches never
  // overlap: they run in order on the one stream of the call that issues them (calls share the workspace, too).
  int* d_tc_sched = nullptr;
  long long* d_tc_dbg = nullptr;   // [256][16] profiling counters of the last tensor-core conv launch
  bool tc_dbg_on = false;
  int fuse_pairs = 1;              // 1 = ResBlock pairs with C <= 64 run in a fused pair kernel (intermediate stays on chip: 8 instead of 20 B of HBM traffic per element pair)
  int pair_ts = 2;                 // form of the fused pair kernel (tc_conv.cu): 2 = 256-row tiles (default), 1 = the same with
                                   // conv2's A operand in registers (register-A wgmma), 0 = 128-row tiles
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  size_t hbm_bytes = 0;
  std::string err;
  int64_t launches = 0;
  cudaStream_t own_stream = nullptr;   // used by the *_host entry points

  // ---- weights (device) ----
  ModelWeights hg;              // HiFiGAN generator
  ModelWeights ac;              // acoustic model
  ModelWeights du;              // duration model (TokenEncoder + projection head)

  // mel filterbank + fft tables
  float* mel_fb = nullptr;      // dense [80][513]
  int* mel_lo = nullptr;        // [80] first non-zero bin
  int* mel_hi = nullptr;        // [80] one past last non-zero bin
  float* fft_tw = nullptr;      // [1024][2] cos/sin(-2 pi k/1024)
  float* hann = nullptr;        // [1024]
  bool fft_ready = false;       // fft_tw and hann uploaded (vtts_fft_tables)
  bool mel_loaded = false;

  // ---- workspace (device), grown on demand ----
  void* ws = nullptr;
  size_t ws_bytes = 0;
  // pinned host staging + device staging for *_host calls
  void* hpin = nullptr;
  size_t hpin_bytes = 0;
  void* dstage = nullptr;
  size_t dstage_bytes = 0;

  // fp32 polyphase filters of the resampler (resample.cu), one per reduced ratio up / down, designed at first use
  struct RsFilter { int up, down; float* taps; };
  std::vector<RsFilter> rs_filters;
  // fp32 K-weighting cascade of the loudness meter (loudness.cu), one per sample rate, designed at first use: the ten
  // biquad coefficients, the segment transitions A^(seg d) (d = 1, 2, 4, 8, 16) and the sub-block transition A^m
  struct LnFilter { int rate; float coef[10]; float seg[5][16]; float blk[16]; };
  std::vector<LnFilter> ln_filters;

  // taps of the last acoustic forward (point into ws)
  float* tap_enc = nullptr; int64_t tap_enc_n = 0;
  float* tap_cond = nullptr; int64_t tap_cond_n = 0;
  float* tap_melpre = nullptr; int64_t tap_melpre_n = 0;

  static constexpr int NSTAGE = 4;   // 0 hifigan, 1 acoustic, 2 melspec, 3 duration
  cudaEvent_t ev0[NSTAGE] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev1[NSTAGE] = {nullptr, nullptr, nullptr, nullptr};
  cudaStream_t ev_stream[NSTAGE] = {nullptr, nullptr, nullptr, nullptr};
  bool ev_valid[NSTAGE] = {false, false, false, false};

  // optional sub-stage timers (vtts_debug_substages): CUDA events recorded between the kernels of a forward call.
  // ids: acoustic 0 start | 1 encoder | 2 upsample | 3 hoisted cond GEMMs | 4 decoder scan | 5 projection | 6 postnet
  //      hifigan  8 start | 9 conv_pre | 10..13 stage 0..3 (ConvTranspose + 3 ResBlocks) | 14 conv_post
  //      teacher  16 start | 17 encoder+upsample | 18 prenet+hoisted GEMMs | 19 zoneout scan | 20 projection+postnet
  static constexpr int NSUB = 24;
  bool sub_on = false;
  cudaEvent_t sub_ev[NSUB] = {};
  bool sub_set[NSUB] = {};
  void sub_mark(int id, cudaStream_t st) {
    if (!sub_on) return;
    if (!sub_ev[id]) cudaEventCreate(&sub_ev[id]);
    cudaEventRecord(sub_ev[id], st);
    sub_set[id] = true;
  }

  int fail(int code, const char* fmt, ...);
  int ensure_ws(size_t bytes);
  int ensure_staging(size_t host_bytes, size_t dev_bytes);
};

extern std::string g_vtts_create_error;

// bump allocator over the context workspace
struct Arena {
  char* base;
  size_t off = 0;
  size_t cap;
  bool measure;  // if true only compute the size
  Arena(void* b, size_t c, bool m) : base((char*)b), cap(c), measure(m) {}
  template <typename T>
  T* take(size_t n) {
    off = (off + 255) & ~size_t(255);
    T* p = measure ? nullptr : (T*)(base + off);
    off += n * sizeof(T);
    return p;
  }
};

// conv1d.cu
int vtts_launch_conv(vtts_ctx* ctx, const ConvLaunch& L, cudaStream_t st);
// ConvProb::bn_inv of an eval BatchNorm: inv[i] = scale[i] * rsqrt(var[i] + 1e-5), n floats, launched on the default
// stream (load time); the caller checks cudaGetLastError
void vtts_bn_inv(const float* scale, const float* var, float* inv, int n);
// tc_conv.cu
// 16-bit elements of one packed N tile: two bf16 planes, or one fp16 plane (f16)
size_t vtts_tc_packed_elems(int k, int Cin, int N, bool f16);
int vtts_tc_pack_weights(vtts_ctx* ctx, const float* w, void* dst, int k, int Cin, int Cout_total, int n0, int N, bool f16);
int vtts_launch_tc_conv(vtts_ctx* ctx, TcLaunch& L, cudaStream_t st);
// fused ResBlock pair (C = 32 or 64): conv1 -> lrelu -> conv2 -> + x with the intermediate kept in shared memory
int vtts_launch_tc_pair(vtts_ctx* ctx, TcPairLaunch& L, cudaStream_t st);
// generic dispatch (acoustic and duration models): runs `L` on the bf16x3 tensor-core path when ctx->precision is 1 or 2
// and packed weights are given (wpk[prob * ntile + tile], ntile = ceil(Cout/256) tiles of width vtts_tc_tile_n(Cout)),
// else on the FP32 path
int vtts_tc_tile_n(int Cout);
int vtts_conv_dispatch(vtts_ctx* ctx, const ConvLaunch& L, void* const* wpk, cudaStream_t st);
// packs every N tile of one conv weight; returns the number of tiles, appends device pointers to `out`
int vtts_tc_pack_conv(vtts_ctx* ctx, const float* w, int k, int Cin, int Cout, bool f16, char*& cursor, std::vector<void*>& out);
size_t vtts_tc_conv_packed_bytes(int k, int Cin, int Cout, bool f16);
// api.cu: weight slots
void vtts_free_weights(ModelWeights& m);
// replaces *store by one zero-filled device allocation holding tensors of n[i] floats, each 256 B aligned
int vtts_alloc_tensors(vtts_ctx* ctx, const std::vector<size_t>& n, float** store, std::vector<float*>& ptrs);
// one entry of a model's packing table: conv weight w[k][Cin][Cout], packed as bf16 hi/lo planes or as one fp16 plane
struct PackSpec { const float* w; int k, Cin, Cout; bool f16 = false; };
// packs every N tile of every entry of `convs` (vtts_tc_pack_conv) into m.wpk and records m.wpk_t / m.tile0
int vtts_pack_convs(vtts_ctx* ctx, ModelWeights& m, const std::vector<PackSpec>& convs);
// hifigan.cu
int vtts_hifigan_prepare(vtts_ctx* ctx);   // derived weights after load
int vtts_hifigan_run(vtts_ctx* ctx, const float* mel, const int32_t* n_frames, int B, int T, float* wav, cudaStream_t st);
size_t vtts_hifigan_ws_bytes(int B, int T);
// nat.cu: the *_run functions carve ctx->ws, which the caller has sized by the matching *_ws_bytes
int vtts_acoustic_prepare(vtts_ctx* ctx);
size_t vtts_acoustic_ws_bytes(int B, int L, int N);
int vtts_acoustic_run(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur,
                      const int32_t* n_frames, const uint8_t* keep, int mode, uint64_t seed, int B, int L, int N,
                      float* mel, cudaStream_t st);
size_t vtts_acoustic_teacher_ws_bytes(int B, int L, int N);
// dropout_mode of a teacher-forced call (0..3; REFERENCE needs B*N*512 < 2^32), checked before any workspace is sized
int vtts_teacher_mode_check(vtts_ctx* ctx, int mode, int B, int N);
int vtts_acoustic_teacher_run(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur,
                              const int32_t* n_frames, const float* mels_in, const uint8_t* keep, const uint8_t* zone, int mode,
                              uint64_t seed, int B, int L, int N, float* mel1, float* mel2, cudaStream_t st);
// pieces of vtts_acoustic_run that the acoustic stream (acoustic_stream.cu) runs on its own:
// the front half (encoder, upsample, hoisted cond projections) into ctx->ws, sized by vtts_acoustic_ws_bytes(B, L, N);
// zc0 / zc1 receive the [B][N][2048] results inside the workspace
int vtts_acoustic_front(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur, const int32_t* n_frames, int B,
                        int L, int N, const float** zc0, const float** zc1, cudaStream_t st);
// output projection melpre = hout . Wo + bo over B rows of T frames (rows at or past len[b] not written)
int vtts_acoustic_project(vtts_ctx* ctx, const float* hout, const int32_t* len, int B, int T, float* melpre, cudaStream_t st);
// postnet + residual over B rows of T frames, frames at or past len[b] read as zero and are not written; q0 / q1 [B][T][512]
int vtts_acoustic_postnet(vtts_ctx* ctx, const float* melpre, const int32_t* len, int B, int T, float* q0, float* q1, float* mel,
                          cudaStream_t st);
// the first n REFERENCE sub-keys of key `seed`, stream-ordered into out[n]
int vtts_ref_subkeys(vtts_ctx* ctx, uint64_t seed, int n, uint2* out, cudaStream_t st);
// the longest token row the upsample kernel takes (the acoustic entry points reject longer ones)
int vtts_acoustic_max_tokens();
// one launch of the resumable decoder scan (decoder_scan_kernel<true>, see DecScanArgs)
struct DecResume {
  const float* zc0;        // [S][zstride][2048]
  const float* zc1;
  const uint8_t* keep;     // MASK: [S][zstride][2][256]
  const uint2* subkeys;    // REFERENCE: [2 * zstride]
  uint64_t seed;
  int mode;
  const int4* rows;        // device [B] (slot, t0, n, -)
  int B, nmax;             // launch rows (<= 128), largest n
  float* state;            // [S][4][512]
  int zstride, hstride;
  float *p1, *p2, *h0, *h1; // [128][256] x2, [2][128][512] x2
  float* hout;             // [B][hstride][1024]
  unsigned int* bar;
};
int vtts_decoder_scan_resume(vtts_ctx* ctx, const DecResume& r, cudaStream_t st);
int vtts_duration_prepare(vtts_ctx* ctx);
size_t vtts_duration_ws_bytes(int B, int L);
// DurationModel.__call__ (model.py:64-70); dur_sec [B][L] seconds, 0 past lengths[b]
int vtts_duration_run(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float* dur_sec,
                      cudaStream_t st);
// resample.cu: frees the context's cached resampling filters
void vtts_resample_free(vtts_ctx* ctx);
// resample.cu: the stream window step shared by the resample and denoise streams.  Per slot s of a window buffer
// win [S][cap]: tbl[2s] = inputs of the previous push (the window tail [tbl[2s], tbl[2s] + K) moves to [0, K)),
// tbl[2s + 1] = new inputs copied from x [S][F] to [K, K + tbl[2s + 1]).  One launch.
int vtts_stream_window_prep(vtts_ctx* ctx, float* win, int cap, int K, const int* tbl, const float* x, int F, int S, cudaStream_t st);
// resample.cu: per-row bounds of resample_kernel, which place a row's buffer in absolute time
struct RsRow {
  long long x0;       // absolute input index of buffer element 0
  long long lo, hi;   // inputs outside [lo, hi) read as zero
  long long m0;       // absolute index of the row's first output
  long long n_calc;   // outputs computed
  long long n_out;    // outputs written (the ones past n_calc as zero)
};
// resample.cu: one resample_kernel launch at out_rate / in_rate (the context's cached filter).  rows == nullptr: the
// one-shot bounds (row b holds n_in[b] or S_in inputs, S_out outputs written); else per-row bounds, max_out the most
// outputs of a row.
int vtts_resample_run(vtts_ctx* ctx, int in_rate, int out_rate, const float* x, long long x_ld, int S_in, const int* n_in,
                      const RsRow* rows, int B, long long S_out, long long max_out, float* y, long long y_ld, cudaStream_t st);
// denoise.cu: per-row bounds of the STFT frame and overlap-add kernels, which place a row's buffers in absolute time
constexpr long long DN_OPEN = 1LL << 60;   // row length not known yet (stream slot before END)
struct DnRow {
  long long x0;       // absolute index of buffer element 0
  long long n;        // row length (DN_OPEN while a stream slot is open)
  long long g0;       // frame held in workspace row 0 of the row
  long long e0;       // absolute index of the first output written
  long long cnt;      // outputs written
  int nfr;            // frames computed
  int copy;           // the outputs are the inputs (a row of <= 512 samples)
};
// denoise.cu: one launch of the overlap-add kernel (denoise_ola_kernel): output t of row b is the sum of the covering
// windowed time frames ws [B][ws_frames][1024] (frame g at row g - g0) in ascending order over the envelope sum w^2, the
// input itself for copy rows, 0 past n.  rows == nullptr: the one-shot bounds (n_in[b] or S samples, S outputs written).
int vtts_denoise_ola(vtts_ctx* ctx, const float* x, long long x_ld, int S, const int* n_in, const DnRow* rows, int B, long long max_out,
                     const float* ws, int ws_frames, float* y, long long y_ld, cudaStream_t st);
// melspec.cu
// twiddles exp(-2 pi i k / 1024) and the periodic Hann window into ctx->fft_tw / ctx->hann (once per context)
int vtts_fft_tables(vtts_ctx* ctx);
int vtts_melspec_prepare(vtts_ctx* ctx);
int vtts_melspec_run(vtts_ctx* ctx, const float* wav, int B, int S, float* mel, cudaStream_t st);

// canonical blob layouts (weights.cu)
struct TensorSpec { const char* name; int64_t n; };
const std::vector<TensorSpec>& vtts_hifigan_specs();
const std::vector<TensorSpec>& vtts_acoustic_specs();
const std::vector<TensorSpec>& vtts_duration_specs();

// indices into ctx->hg.t  (canonical order: pre, ups 0..3, resblocks 0..11 x (c1_0,c1_1,c1_2,c2_0,c2_1,c2_2), post)
namespace hgi {
constexpr int PRE_W = 0, PRE_B = 1;
__host__ __device__ constexpr int UPS_W(int i) { return 2 + 2 * i; }
__host__ __device__ constexpr int UPS_B(int i) { return 3 + 2 * i; }
// resblock n (0..11), which: 0 = convs1, 1 = convs2, m = 0..2
__host__ __device__ constexpr int RB_W(int n, int which, int m) { return 10 + n * 12 + (which * 3 + m) * 2; }
__host__ __device__ constexpr int RB_B(int n, int which, int m) { return RB_W(n, which, m) + 1; }
constexpr int POST_W = 10 + 12 * 12, POST_B = POST_W + 1;
constexpr int COUNT = POST_B + 1;
}  // namespace hgi

// packing table of the generator (ctx->hg.tiles): the 72 ResBlock convs in hgi order, the ConvTranspose output phases
// of the four stages, conv_pre (two N = 256 tiles) as bf16 hi/lo planes; then the same PK_COUNT entries again as fp16
// planes (VTTS_PRECISION_FP16): entry e + PK_COUNT is the fp16 copy of entry e
namespace hgpk {
constexpr int PK_RB(int n, int which, int m) { return n * 6 + which * 3 + m; }
constexpr int PK_UPS(int i, int r) { return i == 0 ? 72 + r : PK_UPS(i - 1, vc::hg_rate(i - 1)) + r; }
constexpr int PK_PRE = PK_UPS(4, 0), PK_COUNT = PK_PRE + 1;
}  // namespace hgpk

// indices into ctx->ac.t
namespace aci {
constexpr int EMBED = 0;
// encoder conv i: w, b, bn_scale, bn_offset, bn_mean, bn_var
__host__ __device__ constexpr int ENC_CONV(int i, int f) { return 1 + i * 6 + f; }
constexpr int ENC_LSTM_F_W = 19, ENC_LSTM_F_B = 20, ENC_LSTM_B_W = 21, ENC_LSTM_B_B = 22;
constexpr int DEC_L0_W = 23, DEC_L0_B = 24, DEC_L1_W = 25, DEC_L1_B = 26;
constexpr int PROJ_W = 27, PROJ_B = 28, PRE1_W = 29, PRE2_W = 30;
// postnet conv i (0..4): w, b [, bn_scale, bn_offset, bn_mean, bn_var for i<4]
__host__ __device__ constexpr int POST_CONV(int i, int f) { return 31 + i * 6 + f; }
constexpr int COUNT = 31 + 4 * 6 + 2;
}  // namespace aci

// indices into ctx->du.t (duration model): the TokenEncoder block has the acoustic model's layout (aci::EMBED ..
// aci::ENC_LSTM_B_B), followed by the projection head hk.Sequential([Linear(256), gelu, Linear(1)]) (model.py:60-62)
namespace dui {
constexpr int FC1_W = 23, FC1_B = 24, FC2_W = 25, FC2_B = 26;
constexpr int COUNT = 27;
}  // namespace dui
