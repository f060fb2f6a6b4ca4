/*
 * viettts_b200.h -- C ABI of the H100-native vietTTS hot path (libviettts_b200.so).
 *
 * The reference (NTT123/vietTTS) has no FFI: its seams for this path are three
 * Python callables.  Each entry point below names the reference interface it
 * replaces (file:line into the reference tree):
 *
 *   vietTTS/hifigan/mel2wave.py:20-41     mel2wave(mel)            -> vtts_mel2wave_host / vtts_hifigan_forward
 *   vietTTS/nat/text2mel.py:61-82         predict_mel(tok, dur)    -> vtts_predict_mel_host / vtts_acoustic_forward
 *   vietTTS/nat/dsp.py:104-128            MelFilter(...)(y)        -> vtts_melspec_host / vtts_melspec
 *   vietTTS/hifigan/mel2wave.py:35-36     pickle.load(hk_hifi)     -> vtts_load_hifigan
 *   vietTTS/nat/text2mel.py:62-71         pickle.load(acoustic)    -> vtts_load_acoustic
 *   vietTTS/nat/text2mel.py:22-34         predict_duration(tokens) -> vtts_predict_duration_host / vtts_duration_forward
 *   vietTTS/nat/text2mel.py:27-28         pickle.load(duration)    -> vtts_load_duration
 *   vietTTS/nat/gta.py:28-41              forward_fn(params, ...)  -> vtts_gta_host / vtts_acoustic_teacher_forward
 *
 * Conventions
 *   - plain C types only; no torch / CUDA types in signatures (`stream` is a
 *     cudaStream_t passed as void*, NULL = default stream).
 *   - every call returns 0 on success or a negative vtts_status; the message is
 *     available from vtts_last_error().  Nothing throws across the ABI.  There is
 *     NO CPU fallback: without a usable sm_90 (H100) device vtts_create fails.
 *   - one context per GPU; a context is not thread-safe; `*_forward` calls are
 *     stream-ordered and asynchronous, `*_host` calls copy H2D/D2H through pinned
 *     staging owned by the context and return after the result is in host memory.
 *   - "dev" pointers are device memory owned by the caller (e.g. torch tensors'
 *     data_ptr()), float32 unless stated, dense row-major in the documented shape.
 *   - tensors are NWC ([batch, time, channels]) exactly like the Haiku models.
 */
#ifndef VIETTTS_B200_H
#define VIETTTS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vtts_ctx vtts_ctx;

typedef enum vtts_status {
  VTTS_OK = 0,
  VTTS_ERR_BAD_ARG = -1,
  VTTS_ERR_CUDA = -2,
  VTTS_ERR_NOT_LOADED = -3,   /* weights for this stage were not loaded */
  VTTS_ERR_NO_DEVICE = -4,    /* no CUDA device / not an sm_90 part */
  VTTS_ERR_OOM = -5,
  VTTS_ERR_NCCL = -6          /* NCCL missing or a collective failed (vtts_broadcast_weights) */
} vtts_status;

/* dropout handling for the prenet (vietTTS/nat/model.py:95-100: dropout is live at inference) and, in the
 * teacher-forced pass, the zoneout of the decoder state (model.py:162-166) */
typedef enum vtts_dropout_mode {
  VTTS_DROPOUT_OFF = 0,     /* deterministic parity mode: no mask, scale 1 */
  VTTS_DROPOUT_MASK = 1,    /* caller supplies uint8 keep-mask [B,N,2,256]; kept values are scaled by 2 */
  VTTS_DROPOUT_SEED = 2,    /* keep bits drawn on device from threefry2x32(key (lo, hi) = seed; b,t,layer,unit) */
  /* the reference's own JAX/Haiku mask stream, drawn on the device.  seed = (rng[0] << 32) | rng[1], the checkpoint's
   * `rng` words; threefry key words k0 = seed >> 32, k1 = (uint32)seed (the opposite word order of SEED).  Classic
   * threefry layout, Haiku next_rng_key() split chain, jax bernoulli bits (viettts_b200/jaxrng.py states the same in numpy).
   *   inference (acoustic_forward, predict_mel / synthesize / tts_host): frame t, prenet layer l draws
   *     bernoulli(sub-key 2t + l, 0.5, [1,256]); every row uses these masks, so row b equals the reference run on row b
   *     alone, independent of B, of the padded N and of its row index.
   *   teacher forced (acoustic_teacher_forward, gta_host): the reference's whole-batch draws -- 6 sub-keys, keep
   *     [B,N,256] x2 at p 0.5, then zoneout [B,N,512] x4 at p 0.1 in state order h0, c0, h1, c1 -- over the call's B rows;
   *     B*N*512 >= 2^32 is rejected.
   * Mask pointers are ignored and may be NULL. */
  VTTS_DROPOUT_REFERENCE = 3
} vtts_dropout_mode;

/* arithmetic of the dense conv contractions (97 % of the FLOPs):
 *   FP32    every product and sum in IEEE fp32 on the FMA pipe (conv1d.cu) -- the strict parity mode
 *   BF16X3  wgmma tensor cores, each fp32 operand split into bf16 hi+lo, three products
 *           (hi*hi + hi*lo + lo*hi) accumulated in fp32 registers (tc_conv.cu); fp32-class accuracy
 *           (waveform L-inf 2e-5 vs float64), no reduced-precision storage anywhere.
 *   FP16    fast mode for the HiFiGAN generator only: its tensor-core convs (conv_pre, the ConvTranspose phases, the 72
 *           ResBlock convs) take each operand as ONE fp16 value (round to nearest, saturated to +-65504, never inf) and
 *           issue one wgmma product instead of three, fp32 accumulate.  Stated tolerance: waveform L-inf <= 3e-3 and RMS
 *           <= 6e-4 against float64 (about 60 dB below the signal), established on synthetic weights; the activation
 *           range of a real checkpoint is not verified.  conv_post, MelFilter and the acoustic, duration, teacher-forced
 *           and GTA paths run exactly as in BF16X3 (their error compounds through the autoregressive scan).  The fused
 *           ResBlock-pair forms other than the default reject this mode with VTTS_ERR_BAD_ARG. */
typedef enum vtts_precision { VTTS_PRECISION_FP32 = 0, VTTS_PRECISION_BF16X3 = 1, VTTS_PRECISION_FP16 = 2 } vtts_precision;

/* ---- library / context ------------------------------------------------------------ */
int vtts_version(void);                                  /* ABI version, currently 1 */
int vtts_create(int device, vtts_ctx** out);
int vtts_destroy(vtts_ctx* ctx);
const char* vtts_last_error(vtts_ctx* ctx);              /* ctx may be NULL: last error of failed create */
int vtts_device_info(vtts_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, int64_t* hbm_bytes);
int vtts_set_precision(vtts_ctx* ctx, int mode);          /* vtts_precision; applies to later forward calls */
int vtts_get_precision(vtts_ctx* ctx);

/* ---- weights --------------------------------------------------------------------------
 * A "blob" is the float32 concatenation of the Haiku-layout tensors in the canonical order
 * listed in INTEGRATION.md (viettts_b200/weights.py builds it from the unchanged pickles).
 * `blob` may be a host or a device pointer (detected); device blobs let rank != 0 load
 * weights received by an NCCL broadcast without a host round trip. */
int64_t vtts_hifigan_blob_floats(void);                  /* 13 926 017 */
int64_t vtts_acoustic_blob_floats(void);                 /* params + BatchNorm eval statistics */
int64_t vtts_duration_blob_floats(void);                 /* TokenEncoder block of the acoustic blob + projection head */
int vtts_load_hifigan(vtts_ctx* ctx, const float* blob, int64_t n_floats);
int vtts_load_acoustic(vtts_ctx* ctx, const float* blob, int64_t n_floats);
int vtts_load_duration(vtts_ctx* ctx, const float* blob, int64_t n_floats);
/* The one collective of the path (SURVEY.md 8e): rank `root` has loaded its weights (vtts_load_*), every other rank
 * receives the same models -- whichever of hifigan / acoustic / duration the root holds -- by ONE grouped ncclBroadcast
 * of the device arenas and derives its packed tensor-core copies locally; no host round trip, nothing on the hot path
 * afterwards.  `nccl_comm` is an ncclComm_t (passed as void*) whose rank on this process's device matches ctx; `is_root`
 * != 0 on the root rank; `stream` a cudaStream_t or NULL.  Replaces the per-process pickle.load of the reference
 * (hifigan/mel2wave.py:35-36, nat/text2mel.py:62-71) on ranks != root.  NCCL is bound with dlopen at the first call
 * (libnccl.so.2 already in the process, else the loader path, else $VTTS_NCCL_LIB); VTTS_ERR_NCCL if that fails. */
int vtts_broadcast_weights(vtts_ctx* ctx, void* nccl_comm, int root, int is_root, void* stream);
/* librosa-style filterbank [80][513] (MelFilter.__init__, dsp.py:107-113) */
int vtts_load_mel_filterbank(vtts_ctx* ctx, const float* fb, int n_mels, int n_bins);

/* ---- device-pointer, stream-ordered entry points ---------------------------------------- */

/* Generator.__call__ (vietTTS/hifigan/model.py:109-125).
 * mel_dev [B,T,80]; n_frames_dev int32 [B] or NULL (= T for every row; rows are zero-padded
 * at their true end, SURVEY H4); wav_dev [B,256*T] (samples past 256*n_frames[b] are 0). */
int vtts_hifigan_forward(vtts_ctx* ctx, const float* mel_dev, const int32_t* n_frames_dev,
                         int B, int T, float* wav_dev, void* stream);

/* AcousticModel.inference (vietTTS/nat/model.py:123-144).
 * tokens_dev int32 [B,L]; lengths_dev int32 [B] or NULL (= L); dur_frames_dev [B,L] durations in
 * FRAMES (seconds*62.5); n_frames_dev int32 [B] or NULL (= N); keep_mask_dev uint8 [B,N,2,256]
 * (mode MASK) or NULL; mel_dev [B,N,80] (rows past n_frames[b] are 0).
 * Row b equals the reference run on row b alone (batch semantics the reference lacks). */
int vtts_acoustic_forward(vtts_ctx* ctx, const int32_t* tokens_dev, const int32_t* lengths_dev,
                          const float* dur_frames_dev, const int32_t* n_frames_dev,
                          const uint8_t* keep_mask_dev, int dropout_mode, uint64_t seed,
                          int B, int L, int N, float* mel_dev, void* stream);

/* AcousticModel.__call__ (vietTTS/nat/model.py:146-169) with is_training=False, the teacher-forced pass gta.py:24-25 runs:
 * mels_in_dev [B,N,80] is the ground-truth mel ALREADY shifted by one frame (gta.py:34-36).  keep_mask_dev uint8
 * [B,N,2,256] prenet keep-masks (kept values x2); zone_mask_dev uint8 [B,N,4,512] zoneout masks in state order
 * (h0, c0, h1, c1), 1 = keep the previous state (Bernoulli(0.1) in the reference, model.py:161-164); modes SEED and
 * REFERENCE draw both on the device, OFF disables both.  mel1 = projection output (may be NULL), mel2 = mel1 + postnet(mel1). */
int vtts_acoustic_teacher_forward(vtts_ctx* ctx, const int32_t* tokens_dev, const int32_t* lengths_dev,
                                  const float* dur_frames_dev, const int32_t* n_frames_dev, const float* mels_in_dev,
                                  const uint8_t* keep_mask_dev, const uint8_t* zone_mask_dev, int dropout_mode, uint64_t seed,
                                  int B, int L, int N, float* mel1_dev_or_null, float* mel2_dev, void* stream);

/* DurationModel.__call__ (vietTTS/nat/model.py:64-70, is_training=False): TokenEncoder -> Linear(256) -> gelu(tanh
 * form, the jax default) -> Linear(1) -> softplus.  tokens_dev int32 [B,L]; lengths_dev int32 [B] or NULL (= L);
 * dur_sec_dev [B,L] predicted durations in SECONDS (0 past lengths[b]).  Row b equals the reference run on row b alone.
 * The silence clip / word-end zeroing of text2mel (text2mel.py:88-97) is host logic (viettts_b200/nat/text2mel.py). */
int vtts_duration_forward(vtts_ctx* ctx, const int32_t* tokens_dev, const int32_t* lengths_dev, int B, int L,
                          float* dur_sec_dev, void* stream);

/* MelFilter.__call__ (vietTTS/nat/dsp.py:115-128). wav_dev [B,S], S % 256 == 0, S >= 512;
 * mel_dev [B,S/256,80]. */
int vtts_melspec(vtts_ctx* ctx, const float* wav_dev, int B, int S, float* mel_dev, void* stream);

/* optional taps for tests: copy an internal activation of the LAST forward call to host.
 * name: "enc" [B,L,512] (of the last acoustic OR duration call), "cond" [B,N,512], "mel_pre" [B,N,80] (before the postnet;
 * after an acoustic stream push: the stream's [max_streams, max_frames, 80] projection outputs, valid for the frames
 * each slot has scanned). */
int vtts_debug_read(vtts_ctx* ctx, const char* name, float* host_out, int64_t n_floats);

/* test hook: one hk.Conv1D (SAME padding, dilation, optional leaky_relu on the input and residual
 * add) on device buffers through any arithmetic path (`precision` a vtts_precision; FP16 packs the weights as the
 * generator's fp16 plane).  x [B,T,Cin], w Haiku layout [k,Cin,Cout],
 * out/resid [B,T,Cout]; len int32 [B] or NULL; pre_slope 1.0 = no input activation.  Synchronous. */
int vtts_debug_conv1d(vtts_ctx* ctx, int precision, const float* x_dev, const float* w_dev, const float* bias_dev,
                      const float* resid_dev, const int32_t* len_dev, int B, int T, int Cin, int Cout, int k, int dil,
                      float pre_slope, float* out_dev);

/* test hook: nprob convs of one shape through the shared conv dispatcher, the path of every acoustic and duration
 * conv and hoisted GEMM (packing, N tiles of <= 256 columns, partial last tile, <= 8 problems per launch, eval BatchNorm
 * and activation epilogue).  Per problem p: x[p] [B,T,Cin], w[p] Haiku layout [k,Cin,Cout], bias[p] [Cout],
 * bn[p] NULL or [4][Cout] (Haiku scale, offset, mean, var), resid[p] NULL or [B,T,Cout], out[p] [B,T,Cout]; host arrays
 * of device pointers (bn and resid may be NULL as a whole).  SAME padding with dilation `dil`; post_act 0 none, 1 tanh,
 * 2 relu, after the BatchNorm and before the residual; len int32 [B] or NULL.  Rows at or past len[b] are not written.
 * `precision` is a vtts_precision (FP16 runs bf16x3 here, as the model does); the context's own mode is left unchanged.
 * Synchronous. */
int vtts_debug_conv_dispatch(vtts_ctx* ctx, int precision, int nprob, const float* const* x, const float* const* w,
                             const float* const* bias, const float* const* bn, const float* const* resid, float* const* out,
                             const int32_t* len, int B, int T, int Cin, int Cout, int k, int dil, int post_act);

/* test hook: one fused ResBlock pair out = conv2(lrelu(conv1(lrelu(x)) + b1)) + b2 + x  (vietTTS/hifigan/model.py:44-51)
 * on the tensor-core path; x/out [B,T,C] with C in {32,64}, w1/w2 Haiku layout [k,C,C], conv1 dilation `dil`. Synchronous.
 * Runs on fp16 operands when the context is in VTTS_PRECISION_FP16, on bf16x3 otherwise. */
int vtts_debug_pair(vtts_ctx* ctx, const float* x_dev, const float* w1_dev, const float* b1_dev, const float* w2_dev,
                    const float* b2_dev, const int32_t* len_dev, int B, int T, int C, int k, int dil, float slope, float* out_dev);

/* test hook: exactly one layer of the generator forward (vtts_hifigan_forward), on caller buffers, with the loaded
 * weights, the context's precision mode and its fused-pair setting; the forward runs the same functions in order.
 * T and n_frames (int32 [B] or NULL) are in mel frames as for the forward; stage i runs on T*S_i rows per batch row
 * with S_0..S_4 = 1, 8, 64, 128, 256, and rows at or past n_frames[b]*S_i read as zero and are not written.
 * x and out are host arrays of device pointers:
 *   layer 0        conv_pre                 x[0] mel [B,T,80]                   -> out[0] [B,T,512]
 *   layer 1        ConvTranspose of stage 0 x[0] conv_pre output [B,T,512]      -> out[0] [B,8T,256]
 *   layer 1+i      ConvTranspose of stage i (i = 1..3): x[0..2] the three ResBlock chains of stage i-1, [B,T*S_i,C_i]
 *                  (lrelu of their mean is the input)                            -> out[0] [B,T*S_{i+1},C_i/2]
 *   layer 5+3i+m   ResBlock step m (0..2) of stage i (0..3), the three chains k = 3, 7, 11 in one launch (two unfused):
 *                  x[j] [B,T*S_{i+1},C_i/2] -> out[j] = x[j] + conv2(lrelu(conv1(lrelu(x[j])))), same shape; out[j]
 *                  must not alias x[j]
 *   layer 17       conv_post                x[0..2] the three chains of stage 3 [B,256T,32] -> out[0] wav [B,256T]
 *                  (tanh applied; zeros past n_frames[b]*256)
 * with C_i = 512 >> i.  Synchronous. */
int vtts_debug_hifigan_layer(vtts_ctx* ctx, int layer, const float* const* x, float* const* out, const int32_t* n_frames, int B,
                             int T);

/* test hook: the masks VTTS_DROPOUT_REFERENCE applies for key `seed`, drawn on the device by the scans' own draw
 * functions, as uint8 (1 = keep).  kind 0: the autoregressive prenet masks [N,2,256] (shared by every row; B ignored);
 * kind 1: the teacher-forced masks, keep [B,N,2,256] followed by zone [B,N,4,512].  Uses the context's workspace
 * (later debug_read taps are invalid).  Synchronous. */
int vtts_debug_dropout_masks(vtts_ctx* ctx, int kind, uint64_t seed, int B, int N, uint8_t* host_out);

/* test hook: the discrete decisions of vtts_pitch_shift for the same arguments, as the device takes them:
 * dec_dev int32 [B][S / 256 + 1][513], for frame t and bin k 1 | (e < 0) << 1 where k is a peak of frame t and e its
 * wrapped phase deviation princarg(theta_t[k] - theta_t-1[k] - 2 pi k H / N) (which side of the princarg cut it took;
 * 0 in frame 0), and 0 elsewhere (no peak, frames past the row's, copied rows).  Runs the analysis and phase kernels of
 * the call.  Stream-ordered; uses the context's workspace. */
int vtts_debug_pitch_decisions(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones,
                               int32_t* dec_dev, void* stream);

/* profiling aid: per-CTA stall counters (SM clocks) of the LAST tensor-core conv launch.
 * Row = CTA, columns: 0 MMA-role total, 1 MMA wait accumulator-free, 2 MMA wait activations, 3 MMA wait
 * weights, 4 weight-producer wait slot, 5 converter wait slot, 6 converter fill, 7 epilogue wait
 * accumulator, 8 epilogue drain.  enable!=0 turns collection on for later launches; the call
 * synchronises, copies (if host_out != NULL) and clears the counters. */
int vtts_debug_tc_stats(vtts_ctx* ctx, int enable, int64_t* host_out_256x16);

/* profiling aid: per-kernel-group times of the LAST forward calls.  enable != 0 switches the event recording on for later
 * calls.  ms_out24 (may be NULL) receives, for every id with both marks recorded, the elapsed ms since the previous
 * id of the same group (0 otherwise); the call synchronises the device.  ids:
 *   acoustic: 1 TokenEncoder, 2 upsample, 3 hoisted cond GEMMs, 4 decoder scan, 5 output projection, 6 postnet
 *   hifigan:  9 conv_pre, 10..13 up-sampling stage 0..3 (ConvTranspose + three ResBlocks), 14 conv_post
 *   teacher-forced pass: 17 encoder + upsample, 18 prenet + hoisted GEMMs, 19 zoneout scan, 20 projection + postnet */
int vtts_debug_substages(vtts_ctx* ctx, int enable, float* ms_out24);

/* ---- streaming generator: push mel frames per stream slot as they arrive ---------------------
 * A vtts_vocoder_stream holds max_streams independent slots.  Each slot carries every generator layer's context
 * between pushes, so a push costs only the frames it brings.  A slot that has received P frames since BEGIN, without
 * END, has emitted max(0, P - D) frames of 256 samples in total (D = vtts_vocoder_stream_lookahead(), the generator's
 * right receptive field rounded up to whole frames); a push with END emits the rest, so the slot emits exactly P frames.
 * The emitted samples, concatenated, are bit-identical to vtts_hifigan_forward of the whole mel in the same precision
 * mode with the fused ResBlock-pair kernel off.  Modes BF16X3 and FP16; FP32 fails with VTTS_ERR_BAD_ARG.
 * Slots are independent: a slot's output equals that stream run alone.  n_new = 0 without flags leaves a slot idle and
 * untouched.  flags: bit0 BEGIN (reset the slot; may be combined with END), bit1 END.  Pushing frames or END to a slot
 * that has not begun, or that has ended, without BEGIN fails with VTTS_ERR_BAD_ARG.  The stream object owns the carried
 * state (device memory that grows with max_streams * max_chunk_frames); each push also uses the context's workspace. */
typedef struct vtts_vocoder_stream vtts_vocoder_stream;
int vtts_vocoder_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_frames, vtts_vocoder_stream** out);
int vtts_vocoder_stream_destroy(vtts_ctx* ctx, vtts_vocoder_stream* vs);
int vtts_vocoder_stream_lookahead(void);                     /* D, in mel frames */
/* mel_dev [S][F][80] (F = max_chunk_frames, rows past n_new[s] ignored); n_new, flags (bit0 BEGIN, bit1 END) and
 * n_out are HOST int32/uint8/int32 arrays of S = max_streams; wav_dev [S][256*(F+D)], slot s gets 256*n_out[s]
 * samples from its start.  Stream-ordered, asynchronous apart from reading the host arrays. */
int vtts_vocoder_stream_push(vtts_ctx* ctx, vtts_vocoder_stream* vs, const float* mel_dev, const int32_t* n_new,
                             const uint8_t* flags, float* wav_dev, int32_t* n_out, void* stream);
/* the same on host buffers mel [S][F][80] and wav [S][256*(F+D)]; returns when wav is written */
int vtts_vocoder_stream_push_host(vtts_ctx* ctx, vtts_vocoder_stream* vs, const float* mel, const int32_t* n_new,
                                  const uint8_t* flags, float* wav, int32_t* n_out);

/* ---- resampling to the caller's output rate ------------------------------------------------------------------
 * (in_rate, out_rate) reduce by their gcd to up / down; both must be positive and up, down <= 1024 (every pair of
 * standard rates reachable from 16 kHz qualifies: 16000 -> 44100 is 441 / 160, 16000 -> 11025 is 441 / 640), else
 * VTTS_ERR_BAD_ARG.  The output is scipy.signal.resample_poly(x, up, down) with its defaults:
 *   half = 10 * max(up, down);  h[k] = up * w[k] / sum(w),  w[k] = fc * sinc(fc * (k - half)) * kaiser(2 * half + 1, 5)[k],
 *   fc = 1 / max(up, down);  y[m] = sum of x[i] * h[m * down + half - i * up] over 0 <= i < n with the index in
 *   [0, 2 * half];  len(y) = ceil(n * up / down).
 * up == down is an exact copy.  The taps are designed in double and rounded to fp32 once (cached in the context per
 * ratio); every output is an fp32 FMA sum in ascending input index, in every vtts_precision mode. */
/* the double-precision filter h[0 .. 2 * half] of the ratio (a single 1.0 when up == down) into taps[capacity] if it
 * fits; returns the tap count, or VTTS_ERR_BAD_ARG.  Needs no device. */
int vtts_resample_filter(int in_rate, int out_rate, double* taps, int capacity);
/* x_dev [B,S_in]; n_in_dev int32 [B] or NULL (= S_in); y_dev [B,S_out] with S_out = ceil(S_in * up / down); outputs
 * past ceil(n_in[b] * up / down) are 0.  Stream-ordered. */
int vtts_resample(vtts_ctx* ctx, const float* x_dev, const int32_t* n_in_dev, int B, int S_in, int in_rate, int out_rate,
                  float* y_dev, void* stream);
/* the same on host buffers */
int vtts_resample_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S_in, int in_rate, int out_rate, float* y);
/* Streaming resampler with max_streams independent slots: each slot carries its filter history (at most
 * 2 * half / up + 1 input samples and a 64-bit position) across pushes, so the outputs a slot emits, concatenated, are
 * bit-identical to vtts_resample of its whole input.  An output is emitted with the first push after which every input
 * it reads has arrived: before END a slot that has received P samples has emitted
 * min(ceil(P * up / down), max(0, floor((P * up - 1 - half) / down) + 1)) outputs; END emits the rest.
 * vtts_resample_stream_lookahead = floor(half / up): how many input samples an output reads past its own time.
 * flags and slot rules as for the vocoder stream: bit0 BEGIN (resets the slot, also an open one; may be combined with
 * END), bit1 END; n_new = 0 without flags leaves a slot idle and untouched; frames or END to a slot that is not open
 * fail with VTTS_ERR_BAD_ARG.  Every push issues the same two launches. */
typedef struct vtts_resample_stream vtts_resample_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer */
int vtts_resample_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int in_rate, int out_rate,
                                vtts_resample_stream** out, int* out_pitch);
int vtts_resample_stream_destroy(vtts_ctx* ctx, vtts_resample_stream* rs);
int vtts_resample_stream_lookahead(int in_rate, int out_rate);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * y_dev [S][out_pitch], slot s gets n_out[s] outputs from its start.  Stream-ordered. */
int vtts_resample_stream_push(vtts_ctx* ctx, vtts_resample_stream* rs, const float* x_dev, const int32_t* n_new,
                              const uint8_t* flags, float* y_dev, int32_t* n_out, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_resample_stream_push_host(vtts_ctx* ctx, vtts_resample_stream* rs, const float* x, const int32_t* n_new,
                                   const uint8_t* flags, float* y, int32_t* n_out);

/* ---- bias denoiser: STFT spectral subtraction of the vocoder's hiss -------------------------------------------------
 * One row x of n samples, strength s >= 0, bias beta[0..512] >= 0 (the WaveGlow / HiFiGAN `Denoiser` convention):
 *   STFT n_fft 1024, hop 256, periodic Hann w, centered frames with reflect padding 512 (torch.stft(center=True,
 *   pad_mode="reflect"), F = n / 256 + 1 frames);  |X| = sqrt(re^2 + im^2);  M' = max(|X| - s beta[k], 0);
 *   Y = X M' / |X| where |X| > 0, else 0;  y = torch.istft(Y, 1024, 256, window=w, center=True, length=n).
 * Rows of n <= 512 samples cannot be reflect-padded and are returned unchanged, bit for bit.  fp32 in every
 * vtts_precision mode; s beta[k] is rounded to fp32 once.  Each frame is transformed on its own, so the bits of an
 * output depend only on the input samples of the frames covering it: the same row gives the same bits alone, in any
 * batch, and through the stream.  The usual bias is vtts_denoise_bias of the generator's output for an all-zero mel
 * [1, 88, 80]. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values are clamped to [0, S]); bias_dev [513]; y_dev [B,S], not x_dev;
 * outputs past n[b] are 0.  strength finite and >= 0, else VTTS_ERR_BAD_ARG.  Stream-ordered; uses the context's
 * workspace (B * (S / 256 + 1) * 4 KiB). */
int vtts_denoise(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, float strength, const float* bias_dev,
                 float* y_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] and the bias values be finite and >= 0 */
int vtts_denoise_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, float strength, const float* bias, float* y);
/* bias_dev[k] = |X_0[k]|, k = 0..512: the magnitude spectrum of frame 0 of the n-sample waveform wav_dev (n > 512),
 * through the denoiser's own frame code.  Stream-ordered. */
int vtts_denoise_bias(vtts_ctx* ctx, const float* wav_dev, int n, float* bias_dev, void* stream);
/* Streaming denoiser with max_streams independent slots, strength and bias (host [513], finite and >= 0) fixed at
 * create: each slot carries the last 2048 input samples and a 64-bit position, so the outputs a slot emits,
 * concatenated, are bit-identical to vtts_denoise of its whole input (rows of <= 512 samples included).  An output t
 * is emitted with the first push after which the frames covering it are final: before END a slot that has received P
 * samples has emitted min(P, 256 * max(0, floor(P / 256) - 3)) outputs; END emits the rest (also with no new samples).
 * vtts_denoise_stream_lookahead() = 1023: how many input samples an output reads past its own time.  flags and slot
 * rules as for the resample stream.  Every push issues the same three launches (window step, frames, overlap-add). */
typedef struct vtts_denoise_stream vtts_denoise_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer (max_chunk_samples + 1023) */
int vtts_denoise_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, float strength, const float* bias,
                               vtts_denoise_stream** out, int* out_pitch);
int vtts_denoise_stream_destroy(vtts_ctx* ctx, vtts_denoise_stream* ds);
int vtts_denoise_stream_lookahead(void);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * y_dev [S][out_pitch], slot s gets n_out[s] outputs from its start.  Stream-ordered. */
int vtts_denoise_stream_push(vtts_ctx* ctx, vtts_denoise_stream* ds, const float* x_dev, const int32_t* n_new,
                             const uint8_t* flags, float* y_dev, int32_t* n_out, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_denoise_stream_push_host(vtts_ctx* ctx, vtts_denoise_stream* ds, const float* x, const int32_t* n_new,
                                  const uint8_t* flags, float* y, int32_t* n_out);

/* ---- pitch shift: a peak-locked phase vocoder on the denoiser's STFT --------------------------------------------------
 * One row x of n samples, a shift of s semitones (finite, in [-12, 12], else VTTS_ERR_BAD_ARG before anything is
 * launched), r = fp32(2^(s / 12)) computed in double (Laroche & Dolson 1999, "New phase-vocoder techniques for
 * pitch-shifting, harmonizing and other exotic effects"):
 *   the STFT of vtts_denoise (X_t[k], k = 0..512); a_t = |X_t|, theta_t = arg X_t (double);
 *   peaks: a_t[k] > a_t[k-1], a_t[k] >= a_t[k+1], a_t[k] > 0, neighbours outside [0, 512] counting as -1; every bin
 *   belongs to its nearest peak (the lower one on a tie);
 *   omega_t[p] = 2 pi p / N + princarg(theta_t[p] - theta_t-1[p] - 2 pi p H / N) / H (2 pi p / N at t = 0);
 *   psi_t(p) = princarg(psi_t-1[p] + H (r - 1) omega_t[p]), psi_t-1[k] the rotation of the peak that owned bin k in
 *   frame t - 1 (0 before frame 0 and in a frame without peaks); princarg(x) = x - 2 pi rint(x / 2 pi); in double;
 *   D_p = rint((r - 1) p); bin k of peak p adds X_t[k] (-1)^D_p e^(i psi_t(p)) to Z_t[k + D_p] (targets outside [0, 512]
 *   dropped, sums in ascending k);  y = the denoiser's inverse and overlap-add of Z.
 * Rows with s == 0 and rows of n <= 512 are returned unchanged, bit for bit.  fp32 in every vtts_precision mode apart
 * from the double phase recurrence.  Each frame is analysed and synthesized on its own and the recurrence runs once per
 * frame in frame order, so a row gives the same bits alone, in any batch, and through the stream. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); semitones HOST float [B]; y_dev [B,S], not x_dev;
 * outputs past n[b] are 0.  Stream-ordered; uses the context's workspace (about 17 KiB per frame of 256 samples). */
int vtts_pitch_shift(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, float* y_dev,
                     void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_pitch_shift_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* semitones, float* y);
/* Streaming pitch shifter with max_streams independent slots: each slot carries the denoise stream's window of 2048
 * inputs and its 64-bit position, the index of its next unscanned frame, theta and psi (double) of the last scanned frame
 * and the synthesized frames later outputs still overlap, so the outputs a slot emits, concatenated, are bit-identical
 * to vtts_pitch_shift of its whole input.  Outputs are released on the denoise stream's schedule (before END
 * min(P, 256 * max(0, floor(P / 256) - 3)) after P samples; END emits the rest) and vtts_pitch_shift_stream_lookahead()
 * = 1023.  A slot's shift is read from semitones[s] with BEGIN and fixed until END.  flags and slot rules as for the
 * resample stream.  Every push issues the same five launches (window step, analysis, phase, synthesis, overlap-add). */
typedef struct vtts_pitch_shift_stream vtts_pitch_shift_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer (max_chunk_samples + 1023) */
int vtts_pitch_shift_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, vtts_pitch_shift_stream** out, int* out_pitch);
int vtts_pitch_shift_stream_destroy(vtts_ctx* ctx, vtts_pitch_shift_stream* ps);
int vtts_pitch_shift_stream_lookahead(void);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * semitones HOST float [S]: read for the slots with BEGIN (finite, in [-12, 12]); for the other pushed slots it must
 * hold the slot's shift, or semitones may be NULL when no slot begins.  y_dev [S][out_pitch], not x_dev, slot s gets
 * n_out[s] outputs from its start.  Argument errors fail with VTTS_ERR_BAD_ARG before anything is launched.
 * Stream-ordered. */
int vtts_pitch_shift_stream_push(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x_dev, const int32_t* n_new,
                                 const uint8_t* flags, const float* semitones, float* y_dev, int32_t* n_out, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_pitch_shift_stream_push_host(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x, const int32_t* n_new,
                                      const uint8_t* flags, const float* semitones, float* y, int32_t* n_out);

/* ---- loudness: ITU-R BS.1770-4 gated loudness and true peak, and normalization to a target ------------------------
 * One mono row x of n samples at rate r, a multiple of 10 in [8000, 192000] (else VTTS_ERR_BAD_ARG):
 *   K-weighting: the libebur128 shelf and high-pass biquads for r, from zero state;  m = r / 10;  E_k = sum of y^2 over
 *   sub-block k (whole sub-blocks only, K = floor(n / m));  blocks j < J = max(0, K - 3):
 *   z_j = (E_j + E_j+1 + E_j+2 + E_j+3) / 4m,  l_j = -0.691 + 10 log10 z_j;  integrated: the mean z over blocks with
 *   l_j > -70 gives Gamma = its loudness - 10, and L = -0.691 + 10 log10(mean z over blocks with l_j > -70 and
 *   l_j > Gamma), -inf with no such block;  momentary l_J-1;  short-term -0.691 + 10 log10(sum of the last 30 E_k / 30m)
 *   (-inf for K < 30);  true peak 20 log10 max(max |x|, max |resample_poly(x, 4, 1)|) dBTP (-inf for silence).
 * fp32 in every vtts_precision mode; each E_k is a fixed function of the filter state entering sub-block k and its
 * samples, and every reduction has an order fixed by the sub-block or block index, so a row gives the same bits alone,
 * in any batch, and through the stream. */
/* coeffs[10] = b0 b1 b2 a1 a2 of the shelf, then of the high-pass, in double (a0 = 1).  Needs no device. */
int vtts_loudness_filter(int rate, double* coeffs);
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); out_dev [B][4] = integrated, momentary and
 * short-term LUFS, true peak dBTP.  Stream-ordered; uses the context's workspace (the 4x oversampled rows, 16 bytes per sample). */
int vtts_loudness(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float* out_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_loudness_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float* out);
/* y = x * fp32(10^(g / 20)) per row, g = target - L, with a ceiling min(g, ceiling - true peak); g = 0 (a bit copy) when
 * L = -inf; outputs past n[b] are 0.  target in [-70, 0] LUFS; ceiling +inf (none) or in [-20, 0] dBTP.  g and the factor
 * are computed on the device (no host synchronisation).  y_dev may equal x_dev; gain_db_dev [B] receives g, or NULL. */
int vtts_loudness_normalize(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float target,
                            float ceiling, float* y_dev, float* gain_db_dev, void* stream);
/* the same on host buffers; gain_db [B] or NULL */
int vtts_loudness_normalize_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float target,
                                 float ceiling, float* y, float* gain_db);
/* Streaming meter with max_streams independent slots: each slot carries the filter state at its last complete
 * sub-block boundary, the samples of the incomplete one, its E_k history (10 * max_seconds sub-blocks), the 4x
 * oversampler's window and the running peak.  After every push a slot's integrated, momentary and short-term values equal
 * vtts_loudness of the samples it has received since BEGIN, bit for bit; its true peak covers the samples and the
 * oversampled outputs whose inputs have all arrived (vtts_loudness_stream_lookahead = 10 samples), and equals the
 * one-shot value after END.  A push that would overflow a slot's history fails with VTTS_ERR_BAD_ARG before anything is
 * launched.  flags and slot rules as for the resample stream; idle and ended slots keep their last readings.  Every push
 * issues the same seven launches. */
typedef struct vtts_loudness_stream vtts_loudness_stream;
int vtts_loudness_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, int max_seconds,
                                vtts_loudness_stream** out);
int vtts_loudness_stream_destroy(vtts_ctx* ctx, vtts_loudness_stream* ls);
int vtts_loudness_stream_lookahead(int rate);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags HOST int32 / uint8 [S]; out_dev [S][4]
 * receives every slot's readings.  Stream-ordered. */
int vtts_loudness_stream_push(vtts_ctx* ctx, vtts_loudness_stream* ls, const float* x_dev, const int32_t* n_new,
                              const uint8_t* flags, float* out_dev, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and out [S][4]; returns when out is written */
int vtts_loudness_stream_push_host(vtts_ctx* ctx, vtts_loudness_stream* ls, const float* x, const int32_t* n_new,
                                   const uint8_t* flags, float* out);

/* ---- streaming acoustic model: every slot advances its decoder a few frames per push ---------------------------
 * A vtts_acoustic_stream holds max_streams (1..128) independent slots.  begin starts utterances in closed slots; each
 * push advances every open slot by min(F, frames left) decoder steps in ONE scan launch and returns the mel frames whose
 * postnet receptive field is complete: after P frames scanned a slot has emitted min(n_emit, max(0, P - D_a)) frames
 * (D_a = vtts_acoustic_stream_lookahead() = 10, the five k = 5 postnet convs), and the push that finishes its scan emits
 * the rest and closes the slot.  A slot scans min(n_frames, n_emit + D_a) frames.  Each utterance's emitted frames,
 * concatenated, are bit-identical to the first n_emit frames of vtts_acoustic_forward of that utterance alone, in the
 * same precision mode (FP32 or BF16X3; FP16 runs as BF16X3) and dropout mode:
 *   OFF; SEED with the slot index as the row (slot s reproduces row s of a call with the same seed); MASK with the
 *   masks given at begin; REFERENCE with the key given at create (the sub-key chain of 2 * max_frames keys is drawn once).
 * Memory: the stream allocates at create, per slot max_frames * (16 KiB zc0 / zc1 + 320 B melpre [+ 512 B MASK keep])
 * + 8 KiB of carried state, plus per-push buffers that grow with max_streams * max_chunk_frames.  max_frames and
 * max_tokens are checked against what vtts_acoustic_forward accepts. */
typedef struct vtts_acoustic_stream vtts_acoustic_stream;
int vtts_acoustic_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_frames, int max_frames, int max_tokens, int dropout_mode,
                                uint64_t seed, vtts_acoustic_stream** out);
int vtts_acoustic_stream_destroy(vtts_ctx* ctx, vtts_acoustic_stream* as);
int vtts_acoustic_stream_lookahead(void);                    /* D_a = 10 mel frames */
/* Start nb utterances (host buffers; synchronous, not on the hot path): slots int32 [nb] distinct closed slots; tokens
 * int32 [nb,L] (L <= max_tokens); lengths int32 [nb] or NULL (= L); dur_frames [nb,L] durations in frames; n_frames
 * int32 [nb] in [1, max_frames]; n_emit int32 [nb] frames to emit, in [1, n_frames], or NULL (= n_frames); keep uint8
 * [nb, max(n_frames), 2, 256] (MASK only, else ignored).  Runs the TokenEncoder, the upsample and the hoisted cond
 * projections of the rows exactly as vtts_acoustic_forward does.  A slot that is still open fails with VTTS_ERR_BAD_ARG. */
int vtts_acoustic_stream_begin(vtts_ctx* ctx, vtts_acoustic_stream* as, int nb, const int32_t* slots, const int32_t* tokens,
                               const int32_t* lengths, const float* dur_frames, const int32_t* n_frames, const int32_t* n_emit,
                               const uint8_t* keep, int L);
/* mel_dev [S][F + D_a][80] (S = max_streams, F = max_chunk_frames): slot s gets n_out[s] frames from its start (rows
 * after them are left as they were); n_out HOST int32 [S], set before anything is launched.  Stream-ordered. */
int vtts_acoustic_stream_push(vtts_ctx* ctx, vtts_acoustic_stream* as, float* mel_dev, int32_t* n_out, void* stream);
/* the same into a host buffer mel [S][F + D_a][80]; returns when it is written */
int vtts_acoustic_stream_push_host(vtts_ctx* ctx, vtts_acoustic_stream* as, float* mel, int32_t* n_out);
/* The duration half of vtts_tts_host for B token rows: predicted durations, silence tokens clipped from below at
 * silence_duration, word-end tokens 0 s, seconds -> frames, the frame count (summed in double, rounded to float, then
 * truncated) and the trailing-silence trim.  Outputs: dur_sec_out [B,L] adjusted seconds (may be NULL); dur_frames_out
 * [B,L] frames (the acoustic model's durations); n_frames_out int32 [B] acoustic frames; n_emit_out int32 [B] frames
 * left after the trim (what vtts_tts_host vocodes, possibly 0). */
int vtts_tts_plan(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float silence_duration, float* dur_sec_out,
                  float* dur_frames_out, int32_t* n_frames_out, int32_t* n_emit_out);

/* ---- host-buffer entry points (what a ctypes / cgo / JNI binding calls) ------------------ */
int vtts_mel2wave_host(vtts_ctx* ctx, const float* mel, const int32_t* n_frames, int B, int T, float* wav);
int vtts_predict_mel_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths,
                          const float* dur_frames, const int32_t* n_frames,
                          const uint8_t* keep_mask, int dropout_mode, uint64_t seed,
                          int B, int L, int N, float* mel);
int vtts_predict_duration_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float* dur_sec);
/* predict_mel -> mel2wave without leaving the device: tokens/durations in, waveform out */
int vtts_synthesize_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths,
                         const float* dur_frames, const int32_t* n_frames,
                         const uint8_t* keep_mask, int dropout_mode, uint64_t seed,
                         int B, int L, int N, float* mel_out_or_null, float* wav);
/* text2mel (vietTTS/nat/text2mel.py:85-103) + mel2wave (synthesizer.py:36-37) for a batch of token rows in one call:
 * predicted durations -> silence tokens clipped from below at silence_duration, word-end tokens 0 s -> frames ->
 * AcousticModel.inference -> trailing-silence frames cut -> Generator.
 * tokens int32 [B,L]; lengths int32 [B] or NULL; dropout_mode OFF, SEED or REFERENCE (MASK is rejected: the frame
 * count is only known inside the call).  Outputs: dur_sec_out [B,L] adjusted
 * durations in seconds (may be NULL); n_frames_out int32 [B] frames of each row's waveform; *n_max_out = row pitch in
 * frames; wav = dense [B][256 * n_max] (samples past 256*n_frames_out[b] are 0), capacity B*256*max_frames floats.
 * If n_max > max_frames nothing is synthesized: the call fails with VTTS_ERR_BAD_ARG after setting *n_max_out and
 * n_frames_out, so the caller can retry with a buffer of that size. */
int vtts_tts_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float silence_duration,
                  int dropout_mode, uint64_t seed, int max_frames, float* dur_sec_out, int32_t* n_frames_out,
                  int32_t* n_max_out, float* wav);
int vtts_melspec_host(vtts_ctx* ctx, const float* wav, int B, int S, float* mel);
/* forward_fn_ of vietTTS/nat/gta.py:28-41 (ground-truth-aligned mels for vocoder fine-tuning): wav_i16 int16 [B,S]
 * (S % 256 == 0) -> /2^15 -> MelFilter -> shift by one frame -> teacher-forced acoustic model -> mel2_out [B,S/256,80].
 * wav_lengths int32 [B] samples or NULL (= S): frames past wav_lengths[b]/256 are 0 (gta.py:74-75 slices them away);
 * dur_sec [B,L] aligned phoneme durations in seconds; masks as in vtts_acoustic_teacher_forward;
 * mel_gt_out_or_null [B,S/256,80] receives the MelFilter output.  Needs vtts_load_acoustic + vtts_load_mel_filterbank. */
int vtts_gta_host(vtts_ctx* ctx, const int16_t* wav_i16, const int32_t* wav_lengths, const int32_t* tokens,
                  const int32_t* lengths, const float* dur_sec, const uint8_t* keep_mask, const uint8_t* zone_mask,
                  int dropout_mode, uint64_t seed, int B, int L, int S, float* mel_gt_out_or_null, float* mel2_out);

/* ---- introspection for bench / tests ------------------------------------------------------ */
/* number of kernel launches issued by this context since creation (our kernels only) */
int64_t vtts_launch_count(vtts_ctx* ctx);
/* elapsed ms of the last forward call of the given stage, measured with CUDA events on the
 * stream the kernels were launched on: stage 0 = hifigan, 1 = acoustic, 2 = melspec, 3 = duration.
 * Synchronises the stream. */
int vtts_last_stage_ms(vtts_ctx* ctx, int stage, float* ms);

#ifdef __cplusplus
}
#endif
#endif /* VIETTTS_B200_H */
