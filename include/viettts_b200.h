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
 *   - the calls on one context run on the device in the order they are issued,
 *     whatever stream each is given: a call waits for the context's previous call
 *     before its first launch (it shares the context's workspace and tile counters),
 *     so a `*_host` call or a push on one stream may follow a `*_forward` call on
 *     another without a synchronisation.  A call issued while its stream captures
 *     a CUDA graph is not ordered this way: order the graph's replays against the
 *     context's other calls on the stream they run on.  Ordering is not thread
 *     safety: calls from several threads still need the caller's lock.
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
 * name: "enc" [B,L,512] (of the last acoustic, teacher-forced OR duration call), "cond" [B,N,512] (autoregressive pass),
 * "mel_pre" [B,N,80] (before the postnet, = mel1 of the teacher-forced pass; after an acoustic stream push: the stream's
 * [max_streams, max_frames, 80] projection outputs, valid for the frames each slot has scanned), "dec_in" [B,N,768]
 * (teacher-forced decoder input [cond | prenet(mels_in)]), "dec_out" [B,N,1024] (decoder scan output [h0 | h1], before
 * zoneout; autoregressive and teacher-forced pass), "dur_hidden" [B,L,256] (duration call: the first Linear's output,
 * bias included, before gelu: the duration head's input; like "enc", unspecified past lengths[b]).  Each call sets
 * every tap, to nothing where it produces none; a call that grows the workspace, and destroying the stream a mel_pre tap points into, clear them all.  Reading a tap
 * that is not set fails with VTTS_ERR_BAD_ARG before any copy. */
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
 * Row = CTA, columns: 0 MMA-role total, 1 epilogue (tc_conv_kernel: after the last wgmma of a tile retires until its
 * outputs are stored), 2 MMA wait activations, 3 MMA wait
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
/* the same on host buffers; n_in[b] must lie in [0, S_in] */
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

/* ---- voice shift: the pitch shift with the formants kept or moved on their own -----------------------------------------
 * vtts_pitch_shift with a formant shift phi per row (finite, in [-12, 12], else VTTS_ERR_BAD_ARG before anything is
 * launched), f = fp32(2^(phi / 12)) computed in double.  Per analysis frame, the real cepstrum of the log magnitudes
 * (floored 80 dB under the frame's peak) liftered to its first 27 coefficients gives the envelope E[k]:
 *   m = max_k a[k];  l[k] = ln max(a[k], 1e-4 m, 1e-30);
 *   c[q] = (l[0] + (-1)^q l[512] + 2 sum_k=1..511 l[k] cos(2 pi k q / 1024)) / 1024, q = 0..26;
 *   E[k] = c[0] + 2 sum_q=1..26 c[q] cos(2 pi k q / 1024).
 * Bin k of peak p, landing on t = k + D_p, is multiplied after its rotation by exp(min(E(t / f) - E[k], ln 10^(24/20))),
 * E(u) linear between E[floor u] and E[floor u + 1] (E[512] past 512), u = t / f in double.  phi = 0 keeps the formants
 * where they are while the pitch moves; phi != 0 moves them by f whatever the pitch does.  Rows with s == 0 and phi == 0,
 * and rows of n <= 512, are copied bit for bit; s == 0 with phi != 0 filters the row's STFT by the gains (r = 1, no phase
 * change).  formants NULL: every row follows the pitch, which is vtts_pitch_shift bit for bit (the vtts_pitch_shift*
 * functions are these calls with formants = NULL).  The envelope is a function of one frame, so a row gives the same bits
 * alone, in any batch, and through the stream. */
/* as vtts_pitch_shift; formants HOST float [B] or NULL.  The workspace grows by 2 KiB per frame of 256 samples. */
int vtts_voice_shift(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* semitones, const float* formants,
                     float* y_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_voice_shift_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* semitones, const float* formants,
                          float* y);
/* vtts_pitch_shift_stream_push with formants HOST float [S] or NULL, on a vtts_pitch_shift_stream: a slot's formant shift
 * is read with BEGIN (NULL: the slots that begin follow the pitch) and fixed until END; for the other pushed slots
 * formants[s] must hold the slot's formant shift, or NaN for a slot that follows the pitch, or formants may be NULL.  A
 * different value for an open slot fails with VTTS_ERR_BAD_ARG before anything is launched.  Schedule, lookahead and
 * launches are the pitch stream's; the outputs a slot emits, concatenated, equal vtts_voice_shift of its whole input. */
int vtts_voice_shift_stream_push(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x_dev, const int32_t* n_new,
                                 const uint8_t* flags, const float* semitones, const float* formants, float* y_dev, int32_t* n_out,
                                 void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_voice_shift_stream_push_host(vtts_ctx* ctx, vtts_pitch_shift_stream* ps, const float* x, const int32_t* n_new,
                                      const uint8_t* flags, const float* semitones, const float* formants, float* y, int32_t* n_out);

/* ---- time stretch: the pitch shifter's phase vocoder with moving analysis frames ------------------------------------
 * One row x of n samples, a tempo alpha (fp32, finite, in [0.5, 2], else VTTS_ERR_BAD_ARG before anything is launched;
 * alpha > 1 is faster), after Laroche & Dolson, "Improved phase vocoder time-scale modification of audio" (IEEE TSAP
 * 7(3), 1999):
 *   M = floor(n / (double)alpha + 0.5) outputs;  T = M / 256 + 1 synthesis frames at hop H = 256;
 *   analysis frame t centred at a_t = min(rint(256 t (double)alpha), n - 1), read with the denoiser's window and its
 *   reflection at 0 and n - 1;  h_t = a_t - a_t-1 (>= 1);  peaks and owners as for vtts_pitch_shift;
 *   omega_t[p] = 2 pi p / N + princarg(theta_t[p] - theta_t-1[p] - 2 pi p h_t / N) / h_t;
 *   psi_t(p) = princarg(psi_t-1[p] + (H - h_t) omega_t[p]), psi_0 = 0, in double;
 *   Y_t[k] = X_t[k] e^(i psi_t(owner_t(k)));  y = the denoiser's inverse and overlap-add of Y over T frames, length M.
 * This is vtts_pitch_shift's recurrence with a per-frame h_t and r = 1.  Rows with alpha == 1 and rows of n <= 512 give
 * their first min(n, M) samples, then zeros up to M (so alpha == 1 is a bit copy).  fp32 in every vtts_precision mode
 * apart from the double phase recurrence; a row gives the same bits alone, in any batch, and through the stream. */
/* M for n samples at `tempo`, or -1 for n < 0 or a tempo outside [0.5, 2].  Needs no device. */
int64_t vtts_time_stretch_length(int64_t n, float tempo);
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); tempo HOST float [B]; y_dev [B,Sy], not x_dev:
 * row b gets its first min(M_b, Sy) outputs, zeros past M_b.  Stream-ordered; uses the context's workspace (about
 * 17 KiB per synthesis frame of the longest row). */
int vtts_time_stretch(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* tempo, float* y_dev, int Sy,
                      void* stream);
/* the same on host buffers x [B,S] and y [B,Sy]; n_in[b] must lie in [0, S] */
int vtts_time_stretch_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const float* tempo, float* y, int Sy);
/* test hook: the discrete decisions of vtts_time_stretch, encoded as vtts_debug_pitch_decisions does:
 * dec_dev int32 [B][T_max][513], T_max = max over b of vtts_time_stretch_length(S, tempo[b]) / 256 + 1.  Stream-ordered;
 * uses the context's workspace. */
int vtts_debug_time_stretch_decisions(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const float* tempo,
                                      int32_t* dec_dev, void* stream);
/* Streaming time stretcher with max_streams independent slots, laid out as the pitch-shift stream (2048 carried inputs
 * and a 64-bit position, the next unscanned frame, theta and psi of the last scanned frame, two halves of synthesized
 * frames), so the outputs a slot emits, concatenated, are bit-identical to vtts_time_stretch of its whole input.
 * Schedule: before END, frame t is scanned once a_t + 512 <= P (P inputs received) and P > 512; after Q frames are
 * scanned the slot has released max(0, 256 Q - 511) outputs, those whose every weighing synthesis frame (256 g <
 * u + 512 <= 256 g + 1023) is synthesized (a slot at tempo 1 releases every input it has received); END releases the
 * rest, up to M.  So n_out is known on the host before launch.  vtts_time_stretch_stream_lookahead() = 1536: before
 * END a slot holding P inputs has released more than P / alpha - 1536 outputs.  A slot's tempo is read from tempo[s] with BEGIN and fixed until END.
 * flags and slot rules as for the resample stream.  Every push issues the same five launches (window step, analysis,
 * phase, synthesis, overlap-add). */
typedef struct vtts_time_stretch_stream vtts_time_stretch_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer (2 * max_chunk_samples + 2048) */
int vtts_time_stretch_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, vtts_time_stretch_stream** out,
                                    int* out_pitch);
int vtts_time_stretch_stream_destroy(vtts_ctx* ctx, vtts_time_stretch_stream* ts);
int vtts_time_stretch_stream_lookahead(void);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * tempo HOST float [S]: read for the slots with BEGIN (finite, in [0.5, 2]); for the other pushed slots it must hold the
 * slot's tempo, or tempo may be NULL when no slot begins.  y_dev [S][out_pitch], not x_dev, slot s gets n_out[s]
 * outputs from its start.  Argument errors fail with VTTS_ERR_BAD_ARG before anything is launched.  Stream-ordered. */
int vtts_time_stretch_stream_push(vtts_ctx* ctx, vtts_time_stretch_stream* ts, const float* x_dev, const int32_t* n_new,
                                  const uint8_t* flags, const float* tempo, float* y_dev, int32_t* n_out, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_time_stretch_stream_push_host(vtts_ctx* ctx, vtts_time_stretch_stream* ts, const float* x, const int32_t* n_new,
                                       const uint8_t* flags, const float* tempo, float* y, int32_t* n_out);

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

/* ---- lookahead true-peak limiter ------------------------------------------------------------------------------------
 * One mono row x of n samples at rate r (a multiple of 10 in [8000, 192000]); pre-gain G dB in [-70, 70]; ceiling C dBTP
 * in [-20, 0], c = 10^(C / 20); lookahead A ms in [1, 20], W = max(1, rint(A r / 1000)); release R ms in [1, 2000],
 * beta = exp(-1000 / (R r)):
 *   v = fp32(10^(G / 20)) x;  u = resample_poly(v, 4, 1);  p[t] = max(|v[t]|, max |u[j]| over j in [4(t - 10),
 *   4(t + 10) + 3] inside [0, 4n));  tau = min(1, c / p) (1 where p = 0);  hold h[t] = min tau[t .. t + W - 1] (tau = 1
 *   past n);  attack a[t] = mean of 1 - h over [t - W + 1, t] (h = 1 before 0; over integers 2^32 (1 - h), rounded up);
 *   release d[t] = max(a[t], beta d[t - 1] + (1 - beta) a[t]);  y = v min(tau, 1 - d);  reduction_db = 20 log10 of the
 *   least applied gain (<= 0).  |y| <= c; rows whose peaks stay under c come back as v bit for bit.
 * fp32 in every vtts_precision mode; every value is a fixed function of the samples and of state at boundaries fixed by
 * absolute sample index, so a row gives the same bits alone, in any batch, and through the stream. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); gain_db_dev float [B] or NULL (0 dB), read on
 * the device (clamped to [-70, 70], non-finite as 0); y_dev [B,S] (may equal x_dev), 0 past n[b]; reduction_db_dev [B]
 * or NULL.  Stream-ordered, no host synchronisation, eight launches; uses the context's workspace (about 28 bytes per
 * sample). */
int vtts_limit(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, const float* gain_db_dev, int B, int S, int rate,
               float ceiling, float lookahead_ms, float release_ms, float* y_dev, float* reduction_db_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] and gain_db[b] in [-70, 70] */
int vtts_limit_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, const float* gain_db, int B, int S, int rate, float ceiling,
                    float lookahead_ms, float release_ms, float* y, float* reduction_db);
/* Loudness normalization that reaches the target under a true-peak ceiling with the limiter instead of lowering the
 * gain: measure L (vtts_loudness), limit x at G = T - L, measure the result L_y, limit x again at G + (T - L_y); G is
 * clamped to [-70, 70] and kept where a reading is -inf (silence: G = 0, y = x).  gain_db_dev [B] receives the final G,
 * or NULL.  All on the device with no host synchronisation, 30 launches; y_dev may equal x_dev. */
int vtts_loudness_normalize_limited(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float target,
                                    float ceiling, float lookahead_ms, float release_ms, float* y_dev, float* gain_db_dev,
                                    void* stream);
/* the same on host buffers; gain_db [B] or NULL */
int vtts_loudness_normalize_limited_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float target,
                                         float ceiling, float lookahead_ms, float release_ms, float* y, float* gain_db);
/* Streaming limiter with max_streams independent slots; ceiling, lookahead and release are fixed at create, a slot's
 * pre-gain is read from gain_db[s] (host, [-70, 70]) at its BEGIN.  Before END sample t is released once sample
 * t + L has arrived, L = vtts_limiter_stream_lookahead(rate, lookahead_ms) = W + 19; END releases the rest.  A slot's
 * outputs, concatenated, equal vtts_limit of its whole input bit for bit.  Each slot carries H = 2W + 64 input samples,
 * the release scan's partial map and d_in of the block holding its next output, and its least gain.  flags and slot
 * rules as for the resample stream.  Every push issues the same nine launches. */
typedef struct vtts_limiter_stream vtts_limiter_stream;
/* *out_pitch = max_chunk_samples + L, the outputs per slot of a push's output buffer */
int vtts_limiter_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float ceiling, float lookahead_ms,
                               float release_ms, vtts_limiter_stream** out, int* out_pitch);
int vtts_limiter_stream_destroy(vtts_ctx* ctx, vtts_limiter_stream* ls);
/* L, or VTTS_ERR_BAD_ARG for a bad rate or lookahead.  Needs no device. */
int vtts_limiter_stream_lookahead(int rate, float lookahead_ms);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, gain_db HOST int32 / uint8 / float [S];
 * y_dev [S][out_pitch]: slot s gets n_out[s] (HOST int32 [S]) outputs from its start; reduction_db_dev [S] receives each
 * slot's reduction over what it has released since BEGIN.  Argument errors fail with VTTS_ERR_BAD_ARG before anything is
 * launched.  Stream-ordered. */
int vtts_limiter_stream_push(vtts_ctx* ctx, vtts_limiter_stream* ls, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                             const float* gain_db, float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream);
/* the same on host buffers x [S][max_chunk_samples], y [S][out_pitch] and reduction_db [S]; returns when they are written */
int vtts_limiter_stream_push_host(vtts_ctx* ctx, vtts_limiter_stream* ls, const float* x, const int32_t* n_new, const uint8_t* flags,
                                  const float* gain_db, float* y, int32_t* n_out, float* reduction_db);

/* ---- equalizer: a cascade of second-order IIR sections -------------------------------------------------------------
 * A filter is sos, HOST float64 [K][6], rows b0 b1 b2 a0 a1 a2 (scipy's layout), 1 <= K <= 8.  For one mono row x of n
 * samples, y = scipy.signal.sosfilt(sos, x) from zero state at sample 0; y is not clipped and outputs past n are 0.
 * Each section, normalized by a0 (a0 != 0), must be finite and strictly stable with every pole radius <= 1 - 1e-6
 * (|a2| < 1, |a1| < 1 + a2); anything else fails with VTTS_ERR_BAD_ARG before anything is launched.
 * Every section runs as the trapezoidal state-variable filter of its bilinear transform, fp32 in every vtts_precision
 * mode; every output is a fixed function of the samples and of the cascade state at boundaries of 1024 samples fixed by
 * absolute sample index, so a row gives the same bits alone, in any batch, and through the stream. */
typedef enum vtts_eq_kind {
  VTTS_EQ_HIGHPASS = 0,   /* Butterworth of `order` 1..8, bilinear prewarped to f0: ceil(order / 2) sections */
  VTTS_EQ_LOWPASS = 1,
  VTTS_EQ_LOWSHELF = 2,   /* RBJ Audio EQ Cookbook shelves, q = the shelf slope S in (0, 1], gain_db in [-24, 24]: 1 section */
  VTTS_EQ_HIGHSHELF = 3,
  VTTS_EQ_PEAKING = 4,    /* RBJ peaking EQ, q in [0.1, 30], gain_db in [-24, 24]: 1 section */
  VTTS_EQ_NOTCH = 5       /* RBJ notch, q in [0.1, 30]: 1 section */
} vtts_eq_kind;
/* sos [8][6] receives *n_sections rows with a0 = 1, designed in double for rate in [8000, 192000] and f0 in
 * [10, 0.45 rate] Hz; parameters a kind does not use are ignored.  VTTS_ERR_BAD_ARG for anything out of range.  Needs
 * no device. */
int vtts_eq_design(int kind, int rate, double f0, double q, double gain_db, int order, double* sos, int* n_sections);
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); y_dev [B,S] (may equal x_dev).  Stream-ordered,
 * no host synchronisation, three launches; uses the context's workspace (128 bytes per 1024 samples). */
int vtts_eq(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, const double* sos, int K, float* y_dev,
            void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_eq_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, const double* sos, int K, float* y);
/* Streaming equalizer with max_streams independent slots; the filter is fixed at create.  Every sample is released by
 * the push that brings it (no lookahead): n_out[s] = n_new[s], and a slot's outputs, concatenated, equal vtts_eq of its
 * whole input bit for bit.  Each slot carries the cascade state at its last complete 1024-sample block boundary and the
 * samples of its incomplete block.  flags and slot rules as for the resample stream.  Every push issues the same four
 * launches. */
typedef struct vtts_eq_stream vtts_eq_stream;
int vtts_eq_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, const double* sos, int K, vtts_eq_stream** out);
int vtts_eq_stream_destroy(vtts_ctx* ctx, vtts_eq_stream* es);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * y_dev [S][max_chunk_samples] (may equal x_dev): slot s gets n_out[s] outputs from its start.  Argument errors fail
 * with VTTS_ERR_BAD_ARG before anything is launched.  Stream-ordered. */
int vtts_eq_stream_push(vtts_ctx* ctx, vtts_eq_stream* es, const float* x_dev, const int32_t* n_new, const uint8_t* flags, float* y_dev,
                        int32_t* n_out, void* stream);
/* the same on host buffers x and y [S][max_chunk_samples]; returns when y is written */
int vtts_eq_stream_push_host(vtts_ctx* ctx, vtts_eq_stream* es, const float* x, const int32_t* n_new, const uint8_t* flags, float* y,
                             int32_t* n_out);

/* ---- feed-forward dynamic range compressor ------------------------------------------------------------------------
 * One mono row x of n samples at rate r (an integer in [8000, 192000]); threshold T dBFS in [-60, 0], ratio R in
 * [1, 20], knee W dB in [0, 24], attack A ms in [0.5, 200], release Rel ms in [5, 5000], makeup M dB in [-24, 24]
 * (anything else, NaN included, fails with VTTS_ERR_BAD_ARG before anything is launched):
 *   L = 20 log10 |x|;  x_L = L - G(L) >= 0 with the soft-knee gain computer G (Giannoulis, Massberg & Reiss 2012,
 *   eq. 4: 0 where 2 (L - T) < -W, (1 - 1/R) (L - T + W/2)^2 / (2W) where 2 |L - T| <= W, (1 - 1/R) (L - T) above);
 *   release y1[t] = max(x_L[t], a_R y1[t - 1] + b_R x_L[t]);  attack y_L[t] = a_A y_L[t - 1] + b_A y1[t] (both from
 *   0), a = fp32(exp(-1000 / (tau r))), b = 1 - a;  y = (x m) 10^(-y_L / 20), m = fp32(10^(M / 20));
 *   reduction_db = -max y_L (<= 0, makeup excluded).  Rows that stay below the knee (and R = 1) come back as x m bit
 *   for bit.
 * fp32 in every vtts_precision mode; every value is a fixed function of the samples and of state at boundaries of 256
 * samples fixed by absolute sample index, so a row gives the same bits alone, in any batch, and through the stream. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); y_dev [B,S] (may equal x_dev), 0 past n[b];
 * reduction_db_dev [B] or NULL.  Stream-ordered, no host synchronisation, six launches; uses the context's workspace
 * (about 0.2 bytes per sample). */
int vtts_compress(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float threshold_db, float ratio,
                  float knee_db, float attack_ms, float release_ms, float makeup_db, float* y_dev, float* reduction_db_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S]; reduction_db [B] or NULL */
int vtts_compress_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float threshold_db, float ratio,
                       float knee_db, float attack_ms, float release_ms, float makeup_db, float* y, float* reduction_db);
/* Streaming compressor with max_streams independent slots; every parameter is fixed at create.  Every sample is released
 * by the push that brings it (no lookahead): n_out[s] = n_new[s], and a slot's outputs, concatenated, equal
 * vtts_compress of its whole input bit for bit.  Each slot carries the partial release and attack maps of the block
 * holding its next sample, that block's entering y1 and y_L, and its largest y_L.  flags and slot rules as for the
 * resample stream.  Every push issues the same six launches. */
typedef struct vtts_compressor_stream vtts_compressor_stream;
int vtts_compressor_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float threshold_db, float ratio,
                                  float knee_db, float attack_ms, float release_ms, float makeup_db, vtts_compressor_stream** out);
int vtts_compressor_stream_destroy(vtts_ctx* ctx, vtts_compressor_stream* cs);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * y_dev [S][max_chunk_samples] (may equal x_dev): slot s gets n_out[s] outputs from its start; reduction_db_dev [S]
 * receives each slot's reduction over what it has released since BEGIN.  Argument errors fail with VTTS_ERR_BAD_ARG
 * before anything is launched.  Stream-ordered. */
int vtts_compressor_stream_push(vtts_ctx* ctx, vtts_compressor_stream* cs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                                float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream);
/* the same on host buffers x and y [S][max_chunk_samples] and reduction_db [S]; returns when they are written */
int vtts_compressor_stream_push_host(vtts_ctx* ctx, vtts_compressor_stream* cs, const float* x, const int32_t* n_new, const uint8_t* flags,
                                     float* y, int32_t* n_out, float* reduction_db);

/* ---- split-band de-esser ------------------------------------------------------------------------------------------
 * One mono row x of n samples at rate r (an integer in [8000, 192000]); crossover freq_hz in [1000, 0.45 r]; threshold,
 * ratio, knee, attack and release as for vtts_compress; range_db in [0, 24] (anything else, NaN included, fails with
 * VTTS_ERR_BAD_ARG before anything is launched):
 *   h = the one second-order Butterworth high-pass section of vtts_eq_design(VTTS_EQ_HIGHPASS, r, freq_hz, order 2)
 *   over x from zero state (the equalizer's filter);  y_L = vtts_compress's detector on L = 20 log10 |h| (no makeup);
 *   y^_L = min(y_L, range_db);  g = 10^(-y^_L / 20);  y = x - (1 - g) h, evaluated as fmaf(g - 1, h, x) where
 *   y^_L > 0 and as x where it is 0: the band below the crossover passes untouched and only the high band is turned
 *   down, by at most range_db.  reduction_db = -max y^_L (<= 0).  Rows whose high band stays below the knee (and
 *   ratio 1, and range 0) come back as x bit for bit.
 * fp32 in every vtts_precision mode; the sidechain keeps the equalizer's 1024-sample blocks and the detector the
 * compressor's 256-sample blocks, both fixed by absolute sample index, so a row gives the same bits alone, in any
 * batch, and through the stream. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); y_dev [B,S] (may equal x_dev), 0 past n[b];
 * reduction_db_dev [B] or NULL.  Stream-ordered, no host synchronisation, nine launches (the equalizer's three, then
 * the compressor's six); uses the context's workspace (about 4.3 bytes per sample). */
int vtts_deess(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, float freq_hz, float threshold_db, float ratio,
               float knee_db, float attack_ms, float release_ms, float range_db, float* y_dev, float* reduction_db_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S]; reduction_db [B] or NULL */
int vtts_deess_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, float freq_hz, float threshold_db, float ratio,
                    float knee_db, float attack_ms, float release_ms, float range_db, float* y, float* reduction_db);
/* Streaming de-esser with max_streams independent slots; every parameter is fixed at create.  Every sample is released by
 * the push that brings it (no lookahead): n_out[s] = n_new[s], and a slot's outputs, concatenated, and its reduction
 * equal vtts_deess of its whole input bit for bit.  Each slot carries the equalizer stream's state (the samples of its
 * incomplete 1024-sample block and the filter state at the block's start) and the compressor stream's (partial maps,
 * entering values, largest y^_L).  flags and slot rules as for the resample stream.  Every push issues the same ten
 * launches (the window step, the equalizer's three, the compressor's six). */
typedef struct vtts_deesser_stream vtts_deesser_stream;
int vtts_deesser_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, float freq_hz, float threshold_db, float ratio,
                               float knee_db, float attack_ms, float release_ms, float range_db, vtts_deesser_stream** out);
int vtts_deesser_stream_destroy(vtts_ctx* ctx, vtts_deesser_stream* ds);
/* as vtts_compressor_stream_push: x_dev, y_dev [S][max_chunk_samples] (y_dev may equal x_dev), n_new, flags, n_out HOST
 * [S], reduction_db_dev [S] each slot's reduction over what it has released since BEGIN.  Stream-ordered. */
int vtts_deesser_stream_push(vtts_ctx* ctx, vtts_deesser_stream* ds, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                             float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream);
/* the same on host buffers x and y [S][max_chunk_samples] and reduction_db [S]; returns when they are written */
int vtts_deesser_stream_push_host(vtts_ctx* ctx, vtts_deesser_stream* ds, const float* x, const int32_t* n_new, const uint8_t* flags,
                                  float* y, int32_t* n_out, float* reduction_db);

/* ---- convolution reverb: a uniformly partitioned overlap-save FIR -------------------------------------------------
 * One mono row x of n samples at rate r (an integer in [8000, 192000]), an impulse response h of L taps (1 <= L <= 5 r,
 * finite) and mix in [0, 1] (anything else, NaN included, fails with VTTS_ERR_BAD_ARG before anything is launched):
 *   c[t] = sum_{i=0}^{min(t, L-1)} h[i] x[t - i]  (causal, from zero state);  y[t] = (1 - mix) x[t] + mix c[t], t < n.
 * The tail past the row's end is not emitted (pad x with zeros to hear it); mix = 0 returns x bit for bit.
 * fp32 in every vtts_precision mode, evaluated as y = fmaf(fp32(mix), c, fp32(1 - mix) x) over 512-sample blocks and
 * partitions fixed by absolute sample index: H_k = FFT-1024 of [h[512k .. 512k + 511], 0 x 512], X_j = FFT-1024 of x
 * over [512 (j - 1), 512 (j + 1)) (zeros before 0 and from n on), and block j of c is samples 512..1023 of
 * irfft(sum_{k <= min(j, K-1)} X_{j-k} H_k), K = ceil(L / 512), each bin summed in ascending k.  So a row gives the same
 * bits alone, in any batch, and through the stream. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); ir_dev [L] on the device (its values are the
 * caller's to check: vtts_reverb_host and the stream check them); y_dev [B,S] (may equal x_dev), 0 past n[b].
 * Stream-ordered, no host synchronisation, four launches (IR spectra, input spectra, multiply-accumulate, inverse and
 * mix); uses the context's workspace: 8 K * 513 bytes for the IR spectra plus about 16 bytes per sample. */
int vtts_reverb(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, const float* ir_dev, int L, float mix,
                float* y_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] and every ir[i] be finite */
int vtts_reverb_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const float* ir, int L, float mix, float* y);
/* Streaming reverb with max_streams independent slots; the IR (host [L]) and mix are fixed at create, where the IR's
 * spectra are computed once.  Each slot carries a window of up to 1023 input samples (its last complete block and the
 * incomplete one) and a frequency-domain delay line, the ring of its last R = K + ceil((max_chunk_samples + 511) / 512) - 1
 * input spectra: S * R * 513 * 8 bytes in all (at 48 kHz with a 1.8 s IR, K = 172, about 0.7 MB per slot plus the
 * chunk's share).  Block j is released with the push after which the slot has received 512 (j + 1) samples: before END
 * a slot that has received p samples has emitted 512 floor(p / 512); END emits the rest (also with no new samples).
 * vtts_reverb_stream_lookahead() = 511.  A slot's outputs, concatenated, equal vtts_reverb of its whole input bit for
 * bit.  flags and slot rules as for the resample stream.  Every push issues the same four launches (window step,
 * input spectra into the ring, multiply-accumulate over the ring, inverse and mix). */
typedef struct vtts_reverb_stream vtts_reverb_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer (max_chunk_samples + 511) */
int vtts_reverb_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, const float* ir, int L, float mix,
                              vtts_reverb_stream** out, int* out_pitch);
int vtts_reverb_stream_destroy(vtts_ctx* ctx, vtts_reverb_stream* rs);
int vtts_reverb_stream_lookahead(void);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * y_dev [S][out_pitch], slot s gets n_out[s] outputs from its start.  Stream-ordered. */
int vtts_reverb_stream_push(vtts_ctx* ctx, vtts_reverb_stream* rs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                            float* y_dev, int32_t* n_out, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_reverb_stream_push_host(vtts_ctx* ctx, vtts_reverb_stream* rs, const float* x, const int32_t* n_new, const uint8_t* flags,
                                 float* y, int32_t* n_out);

/* ---- background bed: a music or ambience bed under the voice, ducked by it ---------------------------------------
 * One mono speech row x of n samples at rate r (an integer in [8000, 192000]) and a bank of K <= 8 beds, each Nb
 * samples at r (0.5 r <= Nb <= 600 r) already at its level: bed k is bank_dev[offsets[k] .. offsets[k] + lengths[k]).
 * duck_db D in [0, 40]; threshold, attack and release as for vtts_compress; fade_in Fi in [0, 5 r], tail Tt in
 * [0, 10 r], xfade C in [0, r] with 2 C < Nb of every bed, offset o in [0, Nb) of every bed, all in samples (anything
 * else, NaN included, fails with VTTS_ERR_BAD_ARG before anything is launched):
 *   y_L = vtts_compress's detector (ratio 20, knee 6 dB) on L = 20 log10 |x|, x = 0 from n on;  y^_L = min(y_L, D);
 *   g = 10^(-y^_L / 20);  bl[t] = b[u], u = (t + o) mod P, P = Nb - C, and for u < C the equal-power seam crossfade
 *   sin(pi u / 2C) b[u] + cos(pi u / 2C) b[P + u];  e[t] = (1 - cos(pi t / Fi)) / 2 for t < Fi (else 1) times
 *   (1 + cos(pi (t - n + 1) / Tt)) / 2 for t >= n (else 1);  y[t] = x[t] + g e bl, evaluated as fmaf(g e, bl, x), for
 *   t < n + Tt;  reduction = -max y^_L (<= 0).  A row with bed index -1 comes back as x bit for bit, without a tail
 *   (reduction 0).
 * fp32 in every vtts_precision mode; the detector keeps the compressor's 256-sample blocks fixed by absolute sample index
 * and the bed and envelopes are functions of that index, so a row gives the same bits alone, in any batch, and through
 * the stream. */
/* x_dev [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); bank_dev on the device, offsets int64 and lengths
 * int32 HOST [K]; bed HOST int32 [B] in [-1, K); y_dev [B][S + tail] (not x_dev), 0 from n[b] + tail (n[b] without a
 * bed); reduction_db_dev [B] or NULL.  Stream-ordered, no host synchronisation: one table copy, the key gather and the
 * compressor's six launches; uses the context's workspace (about 4.3 bytes per sample of S + tail). */
int vtts_bed_mix(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, const float* bank_dev,
                 const long long* offsets, const int32_t* lengths, int K, const int32_t* bed, float duck_db, float threshold_db,
                 float attack_ms, float release_ms, int fade_in, int tail, int xfade, long long offset, float* y_dev,
                 float* reduction_db_dev, void* stream);
/* the same on host buffers x [B,S] and y [B][S + tail] (the bank stays on the device); n_in[b] must lie in [0, S];
 * reduction_db [B] or NULL */
int vtts_bed_mix_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const float* bank_dev,
                      const long long* offsets, const int32_t* lengths, int K, const int32_t* bed, float duck_db, float threshold_db,
                      float attack_ms, float release_ms, int fade_in, int tail, int xfade, long long offset, float* y, float* reduction_db);
/* Streaming bed with max_streams independent slots; the bank and every parameter are fixed at create (bank_dev must stay
 * valid until destroy; offsets and lengths are copied).  No lookahead: a push releases every sample it brings, and the
 * push with END also releases the slot's tail (n_out[s] = n_new[s], + tail with END and a bed).  A slot's bed index is
 * read with BEGIN and kept until END; a push that changes it for an open slot without BEGIN fails.  A slot's outputs,
 * concatenated, and its reduction equal vtts_bed_mix of its whole input bit for bit.  Each slot carries the compressor
 * stream's state.  flags and slot rules as for the resample stream.  Every push issues one table copy, the key gather
 * and the compressor's six launches. */
typedef struct vtts_bed_stream vtts_bed_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer (max_chunk_samples + tail) */
int vtts_bed_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, const float* bank_dev, const long long* offsets,
                           const int32_t* lengths, int K, float duck_db, float threshold_db, float attack_ms, float release_ms, int fade_in,
                           int tail, int xfade, long long offset, vtts_bed_stream** out, int* out_pitch);
int vtts_bed_stream_destroy(vtts_ctx* ctx, vtts_bed_stream* bs);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, bed (each slot's bed index, read where
 * BEGIN is set), n_out HOST [S]; y_dev [S][out_pitch], slot s gets n_out[s] outputs from its start; reduction_db_dev [S]
 * each slot's reduction over what it has released since BEGIN.  Stream-ordered. */
int vtts_bed_stream_push(vtts_ctx* ctx, vtts_bed_stream* bs, const float* x_dev, const int32_t* n_new, const uint8_t* flags, const int32_t* bed,
                         float* y_dev, int32_t* n_out, float* reduction_db_dev, void* stream);
/* the same on host buffers x [S][max_chunk_samples], y [S][out_pitch] and reduction_db [S]; returns when they are written */
int vtts_bed_stream_push_host(vtts_ctx* ctx, vtts_bed_stream* bs, const float* x, const int32_t* n_new, const uint8_t* flags, const int32_t* bed,
                              float* y, int32_t* n_out, float* reduction_db);

/* ---- watermark: a keyed spread-spectrum mark and its batched detector ---------------------------------------------
 * Embed, one mono 16 kHz row x of n samples, a key (any uint64) and a strength eps in [0, 0.3] (anything else, NaN
 * included, fails with VTTS_ERR_BAD_ARG before anything is launched): the denoiser's STFT (n_fft 1024, hop 256, periodic
 * Hann, centered frames with reflect padding), Y_f[k] = X_f[k] (1 + eps c(key, j, k)) for k in [20, 219) (312..3422 Hz),
 * every other bin unchanged, j = floor(f / 4) mod 64, then the denoiser's overlap-add.  c = -1 where the top bit of word 0
 * of threefry2x32(key_lo, key_hi, j, k) is set, else +1.  The pattern repeats every 65536 samples (4.096 s).  Digital
 * silence stays silence; eps = 0 and rows of <= 512 samples return x bit for bit.  fp32 in every vtts_precision mode.
 * Detect, per row and key: resample to 16 kHz (vtts_resample) when rate differs; log power of hop-64 frames whitened by
 * its 9-bin moving mean across frequency; per frame phase q in [0, 16) the sums of groups of 4 hop-256 frames less half
 * of each neighbouring group, folded onto the 64-group period (S_j); z = sum_{j,k} S_j[k] c(key, (j + p) mod 64, k) /
 * sqrt(sum S^2) (0 when that is 0).  Aligned (search = 0): p = q = 0, offset 0.  Search: the largest z over the 1024
 * (p, q) and its offset (1024 p - 64 q) mod 65536, where the row's sample 0 sits in the mark's period at 16 kHz (a crop
 * starting at sample c of a marked row reports c mod 65536).  For audio that does not carry the key, z at one (p, q) is
 * a Rademacher sum: P(z >= tau) <= exp(-tau^2 / 2) whatever the audio, so z >= 5 aligned (3.7e-6) and z >= 6.5 in search
 * (1024 exp(-21.1) = 7e-7) are the library's thresholds.  Rows of <= 512 samples at 16 kHz give z = 0. */
/* x_dev [B,S] at 16 kHz; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); y_dev [B,S] (not x_dev), 0 past
 * n[b].  Stream-ordered, no host synchronisation: two launches (frames, overlap-add), one with eps = 0 (the copy). */
int vtts_watermark(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, uint64_t key, float strength, float* y_dev,
                   void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_watermark_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, uint64_t key, float strength, float* y);
/* Streaming embedder with max_streams independent slots on the denoise stream's window and schedule: before END a slot
 * that has received P samples has emitted min(P, 256 max(0, floor(P / 256) - 3)); END emits the rest.
 * vtts_watermark_stream_lookahead() = 1023.  Key and strength are fixed at create.  A slot's outputs, concatenated, equal
 * vtts_watermark of its whole input bit for bit.  flags and slot rules as for the resample stream; every push is one
 * table copy plus three launches. */
typedef struct vtts_watermark_stream vtts_watermark_stream;
/* *out_pitch receives the outputs per slot of a push's output buffer (max_chunk_samples + 1023) */
int vtts_watermark_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, uint64_t key, float strength,
                                 vtts_watermark_stream** out, int* out_pitch);
int vtts_watermark_stream_destroy(vtts_ctx* ctx, vtts_watermark_stream* ws);
int vtts_watermark_stream_lookahead(void);
/* x_dev [S][max_chunk_samples] (samples past n_new[s] ignored); n_new, flags, n_out HOST int32 / uint8 / int32 [S];
 * y_dev [S][out_pitch], slot s gets n_out[s] outputs from its start.  Stream-ordered. */
int vtts_watermark_stream_push(vtts_ctx* ctx, vtts_watermark_stream* ws, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                               float* y_dev, int32_t* n_out, void* stream);
/* the same on host buffers x [S][max_chunk_samples] and y [S][out_pitch]; returns when y is written */
int vtts_watermark_stream_push_host(vtts_ctx* ctx, vtts_watermark_stream* ws, const float* x, const int32_t* n_new, const uint8_t* flags,
                                    float* y, int32_t* n_out);
/* x_dev [B,S] at `rate` (an integer in [8000, 192000] whose ratio to 16000 the resampler takes); n_dev int32 [B] or
 * NULL; keys_dev uint64 [K] on the device, 1 <= K <= 4096; search 0 (aligned) or not; z_dev float [B][K], offset_dev
 * int32 [B][K].  Stream-ordered, no host synchronisation: three launches (four with the resampler); uses the context's
 * workspace, about 3.2 bytes per 16 kHz sample plus 0.8 MB (search) or 51 KB (aligned) per row. */
int vtts_watermark_detect(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, const uint64_t* keys_dev, int K,
                          int search, float* z_dev, int32_t* offset_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_watermark_detect_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, const uint64_t* keys, int K,
                               int search, float* z, int32_t* offset);

/* ---- wire encodings: PCM-16 and G.711 mu-law / A-law -----------------------------------------------------------
 * Encode, per float32 sample x: v = clip(rint(x * 32767), -32768, 32767), the product in double and rint rounding half
 * to even (NaN gives 0, +-Inf clip): the float -> PCM_16 conversion of libsndfile.  VTTS_ENC_PCM16 stores v as int16;
 * VTTS_ENC_ULAW stores the G.711 mu-law code of v >> 2 and VTTS_ENC_ALAW the G.711 A-law code of v >> 3, one uint8
 * each (the codes of CPython's audioop.lin2ulaw / lin2alaw at width 2).  Decode is the G.711 expansion of a code to
 * int16 (mu-law 0x00 -> -32124), or the int16 itself, divided by 32767 in fp32.  Bit-exact in every vtts_precision
 * mode.  Any other encoding, B outside [1, 65535], S < 1, a null buffer or an output that overlaps the input fails with
 * VTTS_ERR_BAD_ARG before anything is launched. */
typedef enum vtts_encoding { VTTS_ENC_PCM16 = 0, VTTS_ENC_ULAW = 1, VTTS_ENC_ALAW = 2 } vtts_encoding;
/* x_dev float [B,S]; n_dev int32 [B] or NULL (= S; values clamped to [0, S]); y_dev [B,S] int16 (PCM16) or uint8
 * (ULAW, ALAW), the code of 0 past n[b] (0, 0xFF, 0xD5).  Stream-ordered, no host synchronisation: one launch. */
int vtts_encode(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int encoding, void* y_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_encode_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int encoding, void* y);
/* c_dev [B,S] int16 (PCM16) or uint8 codes; n_dev as above; y_dev float [B,S], 0 past n[b].  One launch. */
int vtts_decode(vtts_ctx* ctx, const void* c_dev, const int32_t* n_dev, int B, int S, int encoding, float* y_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S] */
int vtts_decode_host(vtts_ctx* ctx, const void* c, const int32_t* n_in, int B, int S, int encoding, float* y);

/* ---- FLAC: lossless compression of the PCM-16 codes --------------------------------------------------------------
 * A row of n samples becomes a native FLAC stream (RFC 9639, streamable subset): mono, 16 bits, the PCM-16 codes of
 * vtts_encode(VTTS_ENC_PCM16), so a decoder gives those codes back exactly.  "fLaC" and one STREAMINFO block (42
 * bytes: block size, min / max frame size, rate, total samples n, MD5 0 = unknown), then ceil(n / block) frames of fixed
 * blocking, each the cheapest of CONSTANT, FIXED 0..4, LPC 1..12 (Rice-coded residuals) and VERBATIM by exact bit count.
 * oracle/flac_oracle.py is the definition: the bytes are the same in every vtts_precision mode.
 * block: 256, 512, 1024, 2048 or 4096.  rate: any rate a frame header can state (a table rate, kHz <= 255, Hz <= 65535,
 * tens of Hz <= 655350).  A bad block or rate, B outside [1, 65535], S < 0, a pitch below vtts_flac_bound, a null
 * buffer or overlapping buffers fail with VTTS_ERR_BAD_ARG before anything is launched.  S = 0 gives every row the
 * 42-byte header alone. */
/* bytes per row that no output of a row of S samples exceeds (VERBATIM frames with the longest headers); -1 for a
 * bad block or S < 0 */
int64_t vtts_flac_bound(int S, int block);
/* x_dev float [B,S]; n_dev int32 [B] or NULL (= S; clamped to [0, S]); row b's stream goes to y_dev + b * y_pitch
 * (y_pitch >= vtts_flac_bound(S, block)) and its byte count to nbytes_dev[b]; nothing past it is written.  A row of
 * n = 0 gives the 42-byte header only.  Stream-ordered, no host synchronisation: five launches (three when S = 0). */
int vtts_flac_encode(vtts_ctx* ctx, const float* x_dev, const int32_t* n_dev, int B, int S, int rate, int block, uint8_t* y_dev,
                     int64_t y_pitch, int32_t* nbytes_dev, void* stream);
/* the same on host buffers; n_in[b] must lie in [0, S].  One copy of the longest row's byte count from every row
 * comes back, and each row's nbytes[b] bytes go to y + b * y_pitch. */
int vtts_flac_encode_host(vtts_ctx* ctx, const float* x, const int32_t* n_in, int B, int S, int rate, int block, uint8_t* y,
                          int64_t y_pitch, int32_t* nbytes);
/* the 4-bit rate code a frame header gives `rate` (1..14), or -1 for a rate FLAC cannot state */
int vtts_flac_rate_code(int rate);
/* Per-slot FLAC stream on the slot protocol of the sample streams (BEGIN / END flags): max_streams 1..65535 slots,
 * pushes of up to max_chunk_samples (1..2^22) new samples per slot.  A slot carries its P mod block samples that no
 * frame holds yet.  A push emits per slot: with BEGIN the 42-byte stream header (total samples and min / max frame size
 * 0, "unknown"), then the frames its samples complete (after P samples since BEGIN, floor(P / block) frames in all),
 * and with END the short last frame (ceil(P / block) in all).  A slot's bytes, concatenated from BEGIN to END, are the
 * one-shot stream of its samples with those three STREAMINFO fields 0.  *out_bytes: the bytes of a push's output
 * buffer.  Frame numbers past 2^31 - 1 are refused. */
typedef struct vtts_flac_stream vtts_flac_stream;
int vtts_flac_stream_create(vtts_ctx* ctx, int max_streams, int max_chunk_samples, int rate, int block, vtts_flac_stream** out,
                            int64_t* out_bytes);
int vtts_flac_stream_destroy(vtts_ctx* ctx, vtts_flac_stream* fs);
/* x_dev float [S][max_chunk_samples]; n_new, flags host [S]; y_dev uint8 [out_bytes]: every slot's bytes packed one after
 * another from y_dev; tbl_dev int32 [S][2]: each slot's (offset, count) in y_dev.  Stream-ordered, no host
 * synchronisation; buffers must not overlap. */
int vtts_flac_stream_push(vtts_ctx* ctx, vtts_flac_stream* fs, const float* x_dev, const int32_t* n_new, const uint8_t* flags,
                          uint8_t* y_dev, int32_t* tbl_dev, void* stream);
/* the same on host buffers: the table comes back first, then only the bytes the slots produced */
int vtts_flac_stream_push_host(vtts_ctx* ctx, vtts_flac_stream* fs, const float* x, const int32_t* n_new, const uint8_t* flags,
                               uint8_t* y, int32_t* tbl);

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
/* any B: the rows run in launches of at most 128 inside the one call (a row's durations do not depend on the others) */
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
/* Joined utterances: G texts of several sentences each, every sentence one token row, in one call.  Each sentence is
 * planned as vtts_tts_host plans it alone (vtts_tts_plan, one host round trip for all rows) and run through the acoustic
 * model; its first n_emit frames are kept.  A text's kept frames, in sentence order, form one mel row, and the
 * generator runs once over the G rows, so the seams are ordinary context to it.
 * tokens int32 [B,L] sentence rows (B is not limited: the acoustic model runs them in launches of at most 128 rows);
 * lengths int32 [B] or NULL; group_start int32 [G+1]: text g owns rows group_start[g] .. group_start[g+1]-1 (0 first,
 * strictly increasing, B last).  dropout_mode OFF, SEED or REFERENCE (MASK is rejected); in SEED mode the rows of launch
 * c draw with key seed ^ (c * 0x9E3779B97F4A7C15), so row r draws as row r of predict_mel's chunked calls.
 * Outputs: dur_sec_out [B,L] as vtts_tts_host (may be NULL); sent_start_out int32 [B] each sentence's first frame in its
 * text's row (a zero-frame sentence gets the next sentence's start); n_frames_out int32 [G] frames of each text;
 * *n_max_out the row pitch in frames; wav dense [G][256 * n_max] (zero past 256 * n_frames_out[g]), capacity
 * G*256*max_frames floats.  If n_max > max_frames nothing is launched after the plan: the call fails with
 * VTTS_ERR_BAD_ARG after setting the frame outputs, so the caller can retry with that size.  Every bad argument fails
 * before any launch. */
int vtts_tts_joined_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, const int32_t* group_start, int G,
                         float silence_duration, int dropout_mode, uint64_t seed, int max_frames, float* dur_sec_out,
                         int32_t* sent_start_out, int32_t* n_frames_out, int32_t* n_max_out, float* wav);
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
