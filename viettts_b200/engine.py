"""Engine: one libviettts_b200 context per GPU + the host-side plumbing around it.

Host buffers are numpy arrays (the reference's seams take/return numpy / jax
arrays on the host); device buffers are torch tensors used purely as memory
containers (`tensor.data_ptr()` is what crosses the C ABI)."""
from __future__ import annotations

import ctypes as C
import threading
from typing import NamedTuple

import numpy as np

from . import _lib, config, weights

DROPOUT_OFF, DROPOUT_MASK, DROPOUT_SEED, DROPOUT_REFERENCE = 0, 1, 2, 3


def _chunk_seed(seed: int, chunk: int) -> int:
    """Key of the on-device dropout stream for the chunk-th slice of an over-long batch (a distinct 64-bit key per
    chunk: `seed + offset` would alias the next seed's first chunk)."""
    return (int(seed) ^ (chunk * 0x9E3779B97F4A7C15)) & 0xFFFFFFFFFFFFFFFF


def _rng_seed(rng, *others) -> int:
    """The `seed` argument of VTTS_DROPOUT_REFERENCE for a checkpoint `rng` (uint32[2]): (rng[0] << 32) | rng[1].
    `others` are the mask / seed arguments of the same call, which must be None alongside `rng`."""
    if any(o is not None for o in others):
        raise ValueError("rng= selects the reference's own mask stream; it cannot be combined with masks= or seed=")
    w = np.asarray(rng).ravel()
    if w.size != 2 or not np.issubdtype(w.dtype, np.integer):
        raise ValueError(f"rng must hold exactly two integer words (the checkpoint's uint32[2] rng), got {np.asarray(rng).shape}")
    return ((int(w[0]) & 0xFFFFFFFF) << 32) | (int(w[1]) & 0xFFFFFFFF)
PRECISION_FP32, PRECISION_BF16X3, PRECISION_FP16 = 0, 1, 2
PRECISIONS = {"fp32": PRECISION_FP32, "bf16x3": PRECISION_BF16X3, "fp16": PRECISION_FP16}
MAX_ACOUSTIC_ROWS = 128   # rows per vtts_acoustic_forward call (csrc/nat.cu MAX_ROWS)


def resample_ratio(in_rate: int, out_rate: int):
    """(up, down): out_rate / in_rate in lowest terms, as vtts_resample takes it (each must be <= 1024)"""
    from math import gcd
    in_rate, out_rate = int(in_rate), int(out_rate)
    if in_rate <= 0 or out_rate <= 0:
        raise ValueError(f"sample rates must be positive, got {in_rate} -> {out_rate}")
    g = gcd(in_rate, out_rate)
    return out_rate // g, in_rate // g


def resample_length(n: int, in_rate: int, out_rate: int) -> int:
    """ceil(n * up / down): the samples `Engine.resample` makes of n input samples"""
    up, down = resample_ratio(in_rate, out_rate)
    return -(-int(n) * up // down)


DENOISE_BINS = config.N_FFT // 2 + 1   # 513
DENOISE_BIAS_FRAMES = 88                # the all-zero mel [1, 88, 80] the default denoiser bias is taken from


def _strength(s) -> float:
    s = float(s)
    if not (np.isfinite(s) and s >= 0):
        raise ValueError(f"denoise strength must be finite and >= 0, got {s}")
    return s


MAX_SEMITONES = 12.0


def _semitones(v, n: int) -> np.ndarray:
    """float32 [n]: a scalar shift for every row, or one per row, each finite and in [-12, 12]"""
    a = np.asarray(v, np.float32)
    a = np.full(n, a, np.float32) if a.ndim == 0 else np.ascontiguousarray(a.reshape(-1), np.float32)
    if a.shape != (n,):
        raise ValueError(f"semitones: one value or one per row ({n}), got {np.shape(v)}")
    if not (np.all(np.isfinite(a)) and np.all(np.abs(a) <= MAX_SEMITONES)):
        raise ValueError(f"semitones must be finite and lie in [-12, 12], got {v}")
    return a


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()  # torch tensor


def _np(a, dtype, shape=None, what="array"):
    a = np.ascontiguousarray(np.asarray(a), dtype=dtype)
    if shape is not None and tuple(a.shape) != tuple(shape):
        raise ValueError(f"{what}: expected shape {tuple(shape)}, got {tuple(a.shape)}")
    return a


class Engine:
    """A context on one H100.  Not thread-safe (like the C context)."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        self.device = int(device)
        h = _lib.c_ctx()
        rc = self.lib.vtts_create(self.device, C.byref(h))
        if rc != 0:
            msg = self.lib.vtts_last_error(None)
            raise _lib.VttsError(rc, msg.decode() if msg else "?")
        self.h = h
        self._hifigan_key = None
        self._acoustic_key = None
        self._duration_key = None
        self._mel_loaded = False
        self._denoise_bias = None   # default denoiser bias of the loaded generator in the current mode (denoiser_bias)

    def close(self):
        if getattr(self, "h", None):
            self.lib.vtts_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        _lib.check(self.h, rc)

    # ---- info ----
    def device_info(self) -> dict:
        sm, ma, mi, hb = C.c_int(), C.c_int(), C.c_int(), C.c_int64()
        self._ck(self.lib.vtts_device_info(self.h, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(hb)))
        return dict(sm_count=sm.value, cc=(ma.value, mi.value), hbm_bytes=hb.value)

    def launch_count(self) -> int:
        return int(self.lib.vtts_launch_count(self.h))

    def last_stage_ms(self, stage: int) -> float:
        ms = C.c_float()
        self._ck(self.lib.vtts_last_stage_ms(self.h, stage, C.byref(ms)))
        return float(ms.value)

    def set_precision(self, mode) -> None:
        """'fp32' (strict, FMA pipe), 'bf16x3' (wgmma tensor cores, split-bf16, fp32 accumulate; the default) or 'fp16'
        (fast generator: one fp16 product per operand pair, fp32 accumulate, waveform L-inf <= 3e-3 against float64 on
        synthetic weights; every other model runs as in 'bf16x3')."""
        m = PRECISIONS.get(mode, mode)
        self._ck(self.lib.vtts_set_precision(self.h, int(m)))
        self._denoise_bias = None

    def debug_conv1d(self, precision, x_t, w_t, bias_t, k, dil, pre_slope=1.0, resid_t=None, len_t=None):
        """Test hook: one conv layer on torch CUDA tensors through either arithmetic path."""
        import torch
        B, T, Cin = x_t.shape
        Cout = w_t.shape[2]
        out = torch.empty((B, T, Cout), dtype=torch.float32, device=x_t.device)
        m = PRECISIONS.get(precision, precision)
        self._ck(self.lib.vtts_debug_conv1d(self.h, int(m), _ptr(x_t), _ptr(w_t), _ptr(bias_t), _ptr(resid_t), _ptr(len_t),
                                            B, T, Cin, Cout, int(k), int(dil), float(pre_slope), _ptr(out)))
        return out

    POST_ACTS = {"none": 0, "tanh": 1, "relu": 2}

    def debug_conv_dispatch(self, precision, xs, ws, biases, k, dil=1, bns=None, resids=None, post_act="none", len_t=None, outs=None):
        """Test hook: len(xs) convs of one shape through the shared conv dispatcher of the acoustic and duration models,
        on torch CUDA tensors.  xs[p] [B,T,Cin], ws[p] [k,Cin,Cout], biases[p] [Cout], bns[p] None or [4,Cout] (scale,
        offset, mean, var), resids[p] None or [B,T,Cout]; post_act 'none', 'tanh' or 'relu'.  Writes outs[p] [B,T,Cout]
        (allocated when not given) except the rows at or past len_t[b], and returns outs."""
        import torch
        n = len(xs)
        B, T, Cin = xs[0].shape
        Cout = ws[0].shape[2]
        if outs is None:
            outs = [torch.empty((B, T, Cout), dtype=torch.float32, device=xs[0].device) for _ in range(n)]

        def arr(ts):
            return None if ts is None else (C.c_void_p * n)(*[_ptr(t) for t in ts])

        m = PRECISIONS.get(precision, precision)
        self._ck(self.lib.vtts_debug_conv_dispatch(self.h, int(m), n, arr(xs), arr(ws), arr(biases), arr(bns), arr(resids), arr(outs),
                                                   _ptr(len_t), B, T, Cin, Cout, int(k), int(dil), self.POST_ACTS[post_act]))
        return outs

    def debug_pair(self, x_t, w1_t, b1_t, w2_t, b2_t, k, dil, slope=0.1, len_t=None):
        """Test hook: one fused ResBlock pair on torch CUDA tensors (tensor-core path; fp16 operands when the engine is
        in 'fp16', bf16x3 otherwise)."""
        import torch
        B, T, Cc = x_t.shape
        out = torch.empty_like(x_t)
        self._ck(self.lib.vtts_debug_pair(self.h, _ptr(x_t), _ptr(w1_t), _ptr(b1_t), _ptr(w2_t), _ptr(b2_t), _ptr(len_t),
                                          B, T, Cc, int(k), int(dil), float(slope), _ptr(out)))
        return out

    HIFIGAN_LAYERS = 18   # 0 conv_pre, 1..4 ConvTranspose of stage i - 1, 5 + 3i + m ResBlock step (i, m), 17 conv_post

    def debug_hifigan_layer(self, layer, xs, outs, n_frames_t=None, T=None):
        """Test hook (vtts_debug_hifigan_layer): exactly one layer of the generator forward on torch CUDA tensors, with
        the loaded weights, the engine's precision mode and fused-pair setting.  xs: one tensor (layers 0 and 1) or three
        (the chains of a stage), [B, rows, C]; outs: one tensor (three for the ResBlock steps 5..16), written in place
        except the rows at or past n_frames_t[b] times the stage's rows per mel frame.  T (mel frames) defaults to the
        rows of xs[0] divided by the stage's rows per mel frame."""
        scale = [1, 1, 8, 64, 128] + [8] * 3 + [64] * 3 + [128] * 3 + [256] * 3 + [256]
        B, rows = xs[0].shape[:2]
        if T is None:
            T = rows // scale[layer]
        arr = lambda ts: (C.c_void_p * len(ts))(*[_ptr(t) for t in ts])  # noqa: E731
        self._ck(self.lib.vtts_debug_hifigan_layer(self.h, int(layer), arr(xs), arr(outs), _ptr(n_frames_t), int(B), int(T)))
        return outs

    PAIR_KERNELS = {"smem": 0, "tmem": 1, "smem2": 2}

    def set_fused_pairs(self, on: bool, kind: str | None = None):
        """Run the C <= 64 ResBlock pairs in the fused pair kernel (off: two tensor-core conv launches per pair).
        kind selects its form: "smem2" 256-row tiles (the default), "tmem" the same with conv2's A operand in registers
        (register-A wgmma), "smem" 128-row tiles."""
        flags = 0x200 | ((1 if on else 0) << 10)
        if kind is not None:
            flags |= 0x800 | (self.PAIR_KERNELS[kind] << 12)
        self._ck(self.lib.vtts_debug_tc_stats(self.h, flags, None))
        self._denoise_bias = None   # the generator's output (and so the default bias) may change in its last bits

    def tc_stats(self, enable=True):
        """Per-CTA stall counters of the last tensor-core conv launch (see vtts_debug_tc_stats)."""
        out = np.zeros((256, 16), np.int64)
        self._ck(self.lib.vtts_debug_tc_stats(self.h, 1 if enable else 0, _ptr(out)))
        return out

    SUBSTAGES = {1: "acoustic.encoder", 2: "acoustic.upsample", 3: "acoustic.cond_gemm", 4: "acoustic.decoder_scan",
                 5: "acoustic.projection", 6: "acoustic.postnet", 9: "hifigan.conv_pre", 10: "hifigan.stage0", 11: "hifigan.stage1",
                 12: "hifigan.stage2", 13: "hifigan.stage3", 14: "hifigan.conv_post", 17: "teacher.encoder_upsample",
                 18: "teacher.prenet_hoisted_gemm", 19: "teacher.zoneout_scan", 20: "teacher.projection_postnet"}

    def substages(self, enable=True) -> dict:
        """Per-kernel-group device times (ms) of the forward calls since the previous call (vtts_debug_substages);
        `enable` switches the event recording on/off for the following calls."""
        out = np.zeros(24, np.float32)
        self._ck(self.lib.vtts_debug_substages(self.h, 1 if enable else 0, _ptr(out)))
        return {name: float(out[i]) for i, name in self.SUBSTAGES.items() if out[i] > 0}

    # ---- weights ----
    def _load(self, fn, pack, src):
        blob = pack(src) if isinstance(src, dict) else src
        n = int(blob.size if isinstance(blob, np.ndarray) else blob.numel())
        if isinstance(blob, np.ndarray):
            blob = _np(blob, np.float32)
        self._ck(fn(self.h, _ptr(blob), n))

    def load_hifigan(self, params, key=None):
        """params: Haiku-layout dict, a packed float32 numpy blob, or a torch CUDA
        tensor holding the blob (e.g. received through an NCCL broadcast)."""
        self._load(self.lib.vtts_load_hifigan, weights.pack_hifigan, params)
        self._hifigan_key = key if key is not None else object()
        self._denoise_bias = None

    def load_acoustic(self, ckpt, key=None):
        self._load(self.lib.vtts_load_acoustic, weights.pack_acoustic, ckpt)
        self._acoustic_key = key if key is not None else object()

    def load_duration(self, ckpt, key=None):
        """ckpt: the duration checkpoint dict (params/aux), a packed numpy blob, or a torch CUDA tensor."""
        self._load(self.lib.vtts_load_duration, weights.pack_duration, ckpt)
        self._duration_key = key if key is not None else object()

    def broadcast_weights(self, nccl_comm, root: int, is_root: bool, stream=None):
        """vtts_broadcast_weights: the root's loaded models reach every rank's context by one grouped ncclBroadcast.
        `nccl_comm`: an ncclComm_t as ctypes.c_void_p / int (e.g. parallel.NcclComm(...).handle)."""
        self._ck(self.lib.vtts_broadcast_weights(self.h, nccl_comm, int(root), 1 if is_root else 0, stream))
        self._denoise_bias = None
        if not is_root:
            self._hifigan_key = self._acoustic_key = self._duration_key = object()

    def load_mel_filterbank(self, fb=None):
        fb = _np(weights.mel_filterbank() if fb is None else fb, np.float32, (config.MEL_DIM, config.N_FFT // 2 + 1), "filterbank")
        self._ck(self.lib.vtts_load_mel_filterbank(self.h, _ptr(fb), fb.shape[0], fb.shape[1]))
        self._mel_loaded = True

    # ---- host-buffer calls -----------------------------------------------------------
    def mel2wave(self, mel, n_frames=None, out=None) -> np.ndarray:
        """mel f32 [B,T,80] -> wav f32 [B,256T] (Generator.__call__, hifigan/model.py:109-125)."""
        mel = _np(mel, np.float32)
        if mel.ndim != 3 or mel.shape[2] != config.MEL_DIM:
            raise ValueError(f"mel must be [B,T,{config.MEL_DIM}], got {mel.shape}")
        B, T, _ = mel.shape
        nf = None if n_frames is None else _np(n_frames, np.int32, (B,), "n_frames")
        if out is not None and (out.shape != (B, T * config.HOP) or out.dtype != np.float32 or not out.flags.c_contiguous):
            raise ValueError(f"out must be C-contiguous float32 {(B, T * config.HOP)}")
        wav = out if out is not None else np.empty((B, T * config.HOP), np.float32)
        self._ck(self.lib.vtts_mel2wave_host(self.h, _ptr(mel), _ptr(nf), B, T, _ptr(wav)))
        return wav

    # receptive field of the generator in mel frames, one side: conv_pre 3 + ups_0 1 + stage-0 ResBlocks 60/8 +
    # stage 1 60/64 + stage 2 60/128 + stage 3 60/256 + ups/conv_post crumbs = 13.3 (hifigan/model.py:44-51,109-125)
    STREAM_HALO = 16

    def mel2wave_stream(self, mel, chunk_frames: int = 32, halo: int | None = None):
        """Chunked vocoding of ONE utterance for low first-audio latency (SURVEY.md §8f row 4): yields the waveform
        in pieces of `chunk_frames` mel frames.  Each piece is computed from its frames plus `halo` frames of
        context on both sides (recomputed, not carried), so the concatenation equals `mel2wave(mel)` exactly:
        every output sample sees its full receptive field, and samples inside the halo are discarded."""
        mel = _np(mel, np.float32)
        if mel.ndim == 3:
            if mel.shape[0] != 1:
                raise ValueError("mel2wave_stream takes one utterance ([T,80] or [1,T,80])")
            mel = mel[0]
        if mel.ndim != 2 or mel.shape[1] != config.MEL_DIM:
            raise ValueError(f"mel must be [T,{config.MEL_DIM}], got {mel.shape}")
        halo = self.STREAM_HALO if halo is None else int(halo)
        if chunk_frames < 1 or halo < 0:
            raise ValueError("chunk_frames >= 1 and halo >= 0 required")
        T = mel.shape[0]
        for t0 in range(0, T, chunk_frames):
            t1 = min(T, t0 + chunk_frames)
            a, b = max(0, t0 - halo), min(T, t1 + halo)
            wav = self.mel2wave(mel[None, a:b])[0]
            yield wav[(t0 - a) * config.HOP: (t1 - a) * config.HOP]

    def open_vocoder_stream(self, max_streams: int, max_chunk_frames: int) -> "VocoderStream":
        """Stateful streaming generator with `max_streams` independent slots (vtts_vocoder_stream_*): push each slot's
        new mel frames as they arrive and get back every waveform frame whose receptive field is complete.  Each push
        costs only the frames it brings; the emitted audio equals `mel2wave` of the whole mel bit for bit (same
        precision mode, fused pairs off).  Needs the generator weights and the 'bf16x3' or 'fp16' mode."""
        return VocoderStream(self, max_streams, max_chunk_frames)

    def open_acoustic_stream(self, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int, seed=None, rng=None,
                             masks: bool = False) -> "AcousticStream":
        """Streaming acoustic model with `max_streams` (<= 128) independent slots (vtts_acoustic_stream_*): `begin`
        starts utterances in free slots, each `push` advances every open slot by up to `max_chunk_frames` decoder steps
        in one scan launch and returns the mel frames that are final.  Each utterance's frames equal `predict_mel` of
        that utterance alone bit for bit.  Dropout, fixed for the stream: `masks=True` (MASK, masks given to `begin`),
        else `seed` (SEED, slot s draws as row s of `predict_mel(seed=)`), else `rng` (REFERENCE), else off."""
        return AcousticStream(self, max_streams, max_chunk_frames, max_frames, max_tokens, seed=seed, rng=rng, masks=masks)

    def open_tts_stream(self, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int = 1024, seed=None,
                        rng=None, output_rate=None, denoise=None, meter=False, semitones=None) -> "TtsStream":
        """Text-to-speech per slot as a stream: one acoustic stream feeding one vocoder stream, the mel never leaving the
        device.  `begin(slot, tokens)` plans the utterance as `tts` does; each `step()` returns the new audio per slot.
        With fused pairs off a slot's audio equals `tts` of the same tokens bit for bit.  `output_rate`: a resample
        stream follows the vocoder on the device and `step()` returns samples at that rate, equal to `resample` of the
        `tts` audio bit for bit.  `denoise`: a strength; a denoise stream with the default bias (`denoiser_bias()`) sits
        between the vocoder and the resampler, and the audio equals `denoise` of the `tts` audio (then resampled) bit for
        bit.  `semitones`: a pitch-shift stream follows the denoiser (before the resampler) with this shift as every slot's
        default (`begin(..., semitones=)` overrides it per slot), and the audio equals `pitch_shift` of the (denoised)
        `tts` audio bit for bit.  `meter=True`: a loudness meter runs last, on what `step()` returns at the output rate (a
        multiple of 10), and `TtsStream.meter()` gives each stepped slot's readings, read back in the step's one
        synchronisation.  Needs the 'bf16x3' or 'fp16' mode (the vocoder stream has no strict fp32 path)."""
        return TtsStream(self, max_streams, max_chunk_frames, max_frames, max_tokens, seed=seed, rng=rng, output_rate=output_rate,
                         denoise=denoise, meter=meter, semitones=semitones)

    def tts_plan(self, tokens, lengths=None, silence_duration=-1.0):
        """vtts_tts_plan: the duration half of `tts` for token rows [B,L].  Returns (durations in seconds [B,L], durations
        in frames [B,L], acoustic frames n_frames [B], frames kept after the trailing-silence trim n_emit [B])."""
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        sec = np.empty((B, L), np.float32)
        frames = np.empty((B, L), np.float32)
        nf = np.empty(B, np.int32)
        ne = np.empty(B, np.int32)
        self._ck(self.lib.vtts_tts_plan(self.h, _ptr(tokens), _ptr(lens), B, L, float(silence_duration), _ptr(sec), _ptr(frames),
                                        _ptr(nf), _ptr(ne)))
        return sec, frames, nf, ne

    def get_precision(self) -> int:
        return int(self.lib.vtts_get_precision(self.h))

    def _acoustic_args(self, tokens, dur_frames, lengths, n_frames, masks, seed, rng=None):
        ref_seed = None if rng is None else _rng_seed(rng, masks, seed)
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        dur = _np(dur_frames, np.float32, (B, L), "durations")
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        if n_frames is None:
            nf = np.array([int(np.sum(dur[b, : (L if lens is None else lens[b])], dtype=np.float32)) for b in range(B)], np.int32)
        else:
            nf = _np(n_frames, np.int32, (B,), "n_frames")
        N = int(nf.max())
        if N < 1:
            raise ValueError("durations sum to less than one frame")
        if ref_seed is not None:
            return tokens, dur, lens, nf, N, None, DROPOUT_REFERENCE, ref_seed
        if masks is not None:
            mode = DROPOUT_MASK
            masks = _np(masks, np.uint8)
            if masks.shape[0] != B or masks.shape[1] < N or masks.shape[2:] != (2, config.PRENET_DIM):
                raise ValueError(f"masks must be uint8 [B,>=N,2,256], got {masks.shape}")
            masks = np.ascontiguousarray(masks[:, :N])
        elif seed is not None:
            mode = DROPOUT_SEED
        else:
            mode = DROPOUT_OFF
        return tokens, dur, lens, nf, N, masks, mode, int(seed or 0)

    @staticmethod
    def _call_seed(mode, seed, chunk):
        # SEED gives every 128-row chunk its own key; the REFERENCE draws do not depend on the row, so every chunk
        # shares the checkpoint's key
        return seed if mode == DROPOUT_REFERENCE else _chunk_seed(seed, chunk)

    def predict_mel(self, tokens, dur_frames, lengths=None, n_frames=None, masks=None, seed=None, rng=None) -> np.ndarray:
        """AcousticModel.inference for a (ragged) batch: tokens int [B,L], durations in FRAMES
        [B,L] -> mel f32 [B,N,80] with N = max_b n_frames[b] (rows past n_frames[b] are 0).
        Dropout (live at inference in the reference): `masks` uint8 [B,N,2,256] keep-masks,
        else `seed` for the on-device threefry stream, else `rng` (the checkpoint's uint32[2]) for the reference's own
        mask stream drawn on the device (every row gets the masks of the reference run on that row alone), else off."""
        tokens, dur, lens, nf, N, masks, mode, seed = self._acoustic_args(tokens, dur_frames, lengths, n_frames, masks, seed, rng)
        B, L = tokens.shape
        mel = np.empty((B, N, config.MEL_DIM), np.float32)
        for b0 in range(0, B, MAX_ACOUSTIC_ROWS):
            b1 = min(B, b0 + MAX_ACOUSTIC_ROWS)
            sl = slice(b0, b1)
            out = np.empty((b1 - b0, N, config.MEL_DIM), np.float32)
            self._ck(self.lib.vtts_predict_mel_host(
                self.h, _ptr(tokens[sl]), _ptr(None if lens is None else lens[sl]), _ptr(dur[sl]), _ptr(nf[sl]),
                _ptr(None if masks is None else np.ascontiguousarray(masks[sl])), mode, self._call_seed(mode, seed, b0 // MAX_ACOUSTIC_ROWS),
                b1 - b0, L, N, _ptr(out)))
            mel[sl] = out
        return mel

    def predict_duration(self, tokens, lengths=None) -> np.ndarray:
        """DurationModel.__call__ (nat/model.py:64-70) for a (ragged) batch: tokens int [B,L] -> predicted
        durations in SECONDS f32 [B,L] (0 past lengths[b]); row b equals the reference run on row b alone."""
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        out = np.empty((B, L), np.float32)
        for b0 in range(0, B, MAX_ACOUSTIC_ROWS):
            b1 = min(B, b0 + MAX_ACOUSTIC_ROWS)
            o = np.empty((b1 - b0, L), np.float32)
            self._ck(self.lib.vtts_predict_duration_host(
                self.h, _ptr(np.ascontiguousarray(tokens[b0:b1])), _ptr(None if lens is None else np.ascontiguousarray(lens[b0:b1])),
                b1 - b0, L, _ptr(o)))
            out[b0:b1] = o
        return out

    @staticmethod
    def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
        """numpy array backed by page-locked host memory.  Passed as `out=` to synthesize / mel2wave the
        library copies D2H straight into it (no staging copy, no page faults of a fresh array).
        The pinned allocation lives exactly as long as the array (or any view of it)."""
        import weakref
        import torch
        t = torch.empty(tuple(shape), dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True)
        a = t.numpy()
        key = a.ctypes.data
        Engine._pinned_keepalive[key] = t            # the tensor owns the memory ...
        weakref.finalize(a, Engine._pinned_keepalive.pop, key, None)   # ... and is dropped with the array
        return a

    _pinned_keepalive: dict = {}

    def synthesize(self, tokens, dur_frames, lengths=None, n_frames=None, masks=None, seed=None, return_mel=False, out=None, rng=None):
        """predict_mel -> mel2wave with the mel staying on the device.  Returns wav [B,256N]
        (and mel [B,N,80] if return_mel).  `out`: optional preallocated float32 [B,256N] result array
        (ideally from `pinned_empty`); it is validated and written in every path (rows land directly in it).
        In SEED mode row r of a call draws the device stream keyed by (seed, r, frame): an utterance's masks depend on
        its row index, not on the padded frame count of the batch; MASK / OFF / `rng` (REFERENCE) modes are position
        independent."""
        tokens, dur, lens, nf, N, masks, mode, seed = self._acoustic_args(tokens, dur_frames, lengths, n_frames, masks, seed, rng)
        B, L = tokens.shape
        if out is not None and (out.shape != (B, N * config.HOP) or out.dtype != np.float32 or not out.flags.c_contiguous):
            raise ValueError(f"out must be C-contiguous float32 {(B, N * config.HOP)}")
        wav = out if out is not None else np.empty((B, N * config.HOP), np.float32)
        mel = np.empty((B, N, config.MEL_DIM), np.float32) if return_mel else None
        for b0 in range(0, B, MAX_ACOUSTIC_ROWS):
            b1 = min(B, b0 + MAX_ACOUSTIC_ROWS)
            sl = slice(b0, b1)
            # row slices of C-contiguous arrays are contiguous: the library writes straight into the result
            self._ck(self.lib.vtts_synthesize_host(
                self.h, _ptr(tokens[sl]), _ptr(None if lens is None else lens[sl]), _ptr(dur[sl]), _ptr(nf[sl]),
                _ptr(None if masks is None else np.ascontiguousarray(masks[sl])), mode, self._call_seed(mode, seed, b0 // MAX_ACOUSTIC_ROWS),
                b1 - b0, L, N, _ptr(None if mel is None else mel[sl]), _ptr(wav[sl])))
        return (wav, mel) if return_mel else wav

    def tts(self, tokens, lengths=None, silence_duration=-1.0, seed=None, max_frames=None, rng=None):
        """Token rows -> waveforms in ONE library call (vtts_tts_host): duration model, the duration fix-ups of
        text2mel.py:88-97, acoustic model, trailing-silence trim (:99-102) and generator, the mel never leaving
        the device.  tokens int [B,L] (rows padded to L), lengths int [B].  Returns (list of f32 waveforms,
        durations_sec f32 [B,L]).  Dropout: `seed` for the on-device counter stream (keyed by row index), else `rng`
        (the checkpoint's uint32[2]) for the reference's own stream (each row as the reference run on it alone), else off."""
        ref_seed = None if rng is None else _rng_seed(rng, seed)
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2:
            raise ValueError("tokens must be [B,L]")
        B, L = tokens.shape
        if B > MAX_ACOUSTIC_ROWS:
            raise ValueError(f"tts: at most {MAX_ACOUSTIC_ROWS} rows per call")
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        dur = np.empty((B, L), np.float32)
        nf = np.zeros(B, np.int32)
        nmax = C.c_int32(0)
        cap = int(max_frames) if max_frames else max(16, int(L * 0.12 * config.SAMPLE_RATE / config.HOP))
        mode = DROPOUT_SEED if seed is not None else DROPOUT_OFF
        if ref_seed is not None:
            mode, seed = DROPOUT_REFERENCE, ref_seed
        for _ in range(2):
            wav = np.empty(B * cap * config.HOP, np.float32)
            rc = self.lib.vtts_tts_host(self.h, _ptr(tokens), _ptr(lens), B, L, float(silence_duration), mode, int(seed or 0),
                                        cap, _ptr(dur), _ptr(nf), C.byref(nmax), _ptr(wav))
            if rc == 0 or not (0 < cap < nmax.value):
                break
            cap = int(nmax.value)       # buffer too small: the call reported the size it needs
        self._ck(rc)
        n = int(nmax.value)
        wav = wav[: B * n * config.HOP].reshape(B, n * config.HOP)
        return [wav[b, : int(nf[b]) * config.HOP].copy() for b in range(B)], dur

    def synthesize_many(self, utterances, seed=None, masks=None, max_pad_frac=0.08, max_rows=32, rng=None):
        """Mixed-length workload (BASELINE configs[4]): `utterances` is a list of (tokens list[int],
        durations_in_frames f32[L]).  They are bucketed by frame count so that padding stays below
        `max_pad_frac`, each bucket runs as one ragged batch, and the waveforms come back in input order
        (list of np.float32 [256*n_frames_i]).  Row i of any bucket equals utterance i run alone (with `rng`, the
        reference's own dropout stream, that includes its masks)."""
        from .parallel import bucket_by_length
        if rng is not None:
            _rng_seed(rng, masks, seed)
        nfs = [int(np.sum(np.asarray(d, np.float32), dtype=np.float32)) for _, d in utterances]
        out = [None] * len(utterances)
        for bucket in bucket_by_length(nfs, max_pad_frac, max_rows):
            Lmax = max(len(utterances[i][0]) for i in bucket)
            tok = np.zeros((len(bucket), Lmax), np.int32)
            dur = np.zeros((len(bucket), Lmax), np.float32)
            lens = np.zeros(len(bucket), np.int32)
            for r, i in enumerate(bucket):
                t, d = utterances[i]
                tok[r, : len(t)] = t
                dur[r, : len(t)] = d
                lens[r] = len(t)
            nf = np.asarray([nfs[i] for i in bucket], np.int32)
            m = None if masks is None else np.stack([np.asarray(masks[i])[: nf.max()] if np.asarray(masks[i]).shape[0] >= nf.max()
                                                     else np.pad(np.asarray(masks[i]), ((0, nf.max() - np.asarray(masks[i]).shape[0]), (0, 0), (0, 0)))
                                                     for i in bucket])
            wav = self.synthesize(tok, dur, lengths=lens, n_frames=nf, masks=m, seed=seed, rng=rng)
            for r, i in enumerate(bucket):
                out[i] = wav[r, : nfs[i] * config.HOP].copy()
        return out

    def _tf_masks(self, B, N, keep_masks, zone_masks, seed, rng=None):
        """(keep, zone, mode, seed) of a teacher-forced call."""
        if rng is not None:
            return None, None, DROPOUT_REFERENCE, _rng_seed(rng, keep_masks, zone_masks, seed)
        if keep_masks is not None or zone_masks is not None:
            if keep_masks is None or zone_masks is None:
                raise ValueError("keep_masks and zone_masks must be given together")
            km = _np(keep_masks, np.uint8, (B, N, 2, config.PRENET_DIM), "keep_masks")
            zm = _np(zone_masks, np.uint8, (B, N, 4, config.ACOUSTIC_DECODER_DIM), "zone_masks")
            return km, zm, DROPOUT_MASK, 0
        return None, None, (DROPOUT_SEED if seed is not None else DROPOUT_OFF), int(seed or 0)

    def teacher_forced(self, tokens, dur_frames, mels_in, lengths=None, n_frames=None, keep_masks=None, zone_masks=None, seed=None,
                       rng=None):
        """AcousticModel.__call__ (nat/model.py:146-169, is_training=False): tokens int [B,L], durations in frames
        [B,L], mels_in f32 [B,N,80] (ground truth shifted by one frame) -> (mel1, mel2) f32 [B,N,80].
        keep_masks uint8 [B,N,2,256] / zone_masks uint8 [B,N,4,512] (1 = keep previous state), else `seed` for the
        on-device stream, else `rng` (the checkpoint's uint32[2]) for the reference's own whole-batch draws on the
        device (= jaxrng.teacher_forced_masks(rng, B, N)), else both off.  Host buffers; the device work is
        vtts_acoustic_teacher_forward."""
        import torch
        tokens = _np(tokens, np.int32)
        B, L = tokens.shape
        mels_in = _np(mels_in, np.float32)
        N = mels_in.shape[1]
        if mels_in.shape != (B, N, config.MEL_DIM):
            raise ValueError(f"mels_in must be [B,N,{config.MEL_DIM}]")
        if B > MAX_ACOUSTIC_ROWS:
            raise ValueError(f"teacher_forced: at most {MAX_ACOUSTIC_ROWS} rows per call")
        km, zm, mode, seed = self._tf_masks(B, N, keep_masks, zone_masks, seed, rng)
        dev = torch.device("cuda", self.device)
        up = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        t_tok, t_dur, t_in = up(tokens), up(_np(dur_frames, np.float32, (B, L), "durations")), up(mels_in)
        t_len = up(None if lengths is None else _np(lengths, np.int32, (B,), "lengths"))
        t_nf = up(None if n_frames is None else _np(n_frames, np.int32, (B,), "n_frames"))
        t_km, t_zm = up(km), up(zm)
        m1 = torch.empty((B, N, config.MEL_DIM), dtype=torch.float32, device=dev)
        m2 = torch.empty_like(m1)
        st = torch.cuda.current_stream(dev).cuda_stream
        self._ck(self.lib.vtts_acoustic_teacher_forward(self.h, _ptr(t_tok), _ptr(t_len), _ptr(t_dur), _ptr(t_nf), _ptr(t_in), _ptr(t_km),
                                                        _ptr(t_zm), mode, seed, B, L, N, _ptr(m1), _ptr(m2), st))
        torch.cuda.synchronize(dev)
        return m1.cpu().numpy(), m2.cpu().numpy()

    def gta(self, wav_i16, tokens, dur_sec, lengths=None, wav_lengths=None, keep_masks=None, zone_masks=None, seed=None, return_gt=False,
            rng=None):
        """forward_fn of nat/gta.py:28-44 in one library call: int16 wavs [B,S] + aligned phonemes -> mel2_hat
        f32 [B,S/256,80] (rows past wav_lengths[b]//256 are 0).  Masks as in `teacher_forced`."""
        if not self._mel_loaded:
            self.load_mel_filterbank()
        wav = np.ascontiguousarray(np.asarray(wav_i16))
        if wav.dtype != np.int16 or wav.ndim != 2:
            raise ValueError("wav_i16 must be int16 [B,S]")
        B, S = wav.shape
        tokens = _np(tokens, np.int32)
        if tokens.ndim != 2 or tokens.shape[0] != B:
            raise ValueError("tokens must be [B,L]")
        L = tokens.shape[1]
        if B > MAX_ACOUSTIC_ROWS:
            raise ValueError(f"gta: at most {MAX_ACOUSTIC_ROWS} rows per call")
        N = S // config.HOP
        km, zm, mode, seed = self._tf_masks(B, N, keep_masks, zone_masks, seed, rng)
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        wl = None if wav_lengths is None else _np(wav_lengths, np.int32, (B,), "wav_lengths")
        gt = np.empty((B, N, config.MEL_DIM), np.float32) if return_gt else None
        out = np.empty((B, N, config.MEL_DIM), np.float32)
        self._ck(self.lib.vtts_gta_host(self.h, _ptr(wav), _ptr(wl), _ptr(tokens), _ptr(lens), _ptr(_np(dur_sec, np.float32, (B, L), "durations")),
                                        _ptr(km), _ptr(zm), mode, seed, B, L, S, _ptr(gt), _ptr(out)))
        return (out, gt) if return_gt else out

    def melspec(self, wav) -> np.ndarray:
        """MelFilter.__call__ (nat/dsp.py:115-128): wav f32 [B,S] -> log-mel [B,S/256,80]."""
        if not self._mel_loaded:
            self.load_mel_filterbank()
        wav = _np(wav, np.float32)
        assert wav.ndim == 2, "MelFilter expects [B,S] (dsp.py:118)"
        B, S = wav.shape
        mel = np.empty((B, S // config.HOP, config.MEL_DIM), np.float32)
        self._ck(self.lib.vtts_melspec_host(self.h, _ptr(wav), B, S, _ptr(mel)))
        return mel

    def debug_read(self, name: str, shape) -> np.ndarray:
        out = np.empty(shape, np.float32)
        self._ck(self.lib.vtts_debug_read(self.h, name.encode(), _ptr(out), out.size))
        return out

    # ---- device-pointer calls (torch tensors as memory containers) --------------------
    def hifigan_forward(self, mel_t, n_frames_t=None, out=None, stream=None):
        import torch
        assert mel_t.is_cuda and mel_t.dtype == torch.float32 and mel_t.is_contiguous()
        B, T, _ = mel_t.shape
        if out is None:
            out = torch.empty((B, T * config.HOP), dtype=torch.float32, device=mel_t.device)
        st = torch.cuda.current_stream(mel_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_hifigan_forward(self.h, _ptr(mel_t), _ptr(n_frames_t), B, T, _ptr(out), st))
        return out

    def debug_dropout_masks(self, kind, rng, B, N) -> np.ndarray:
        """Test hook (vtts_debug_dropout_masks): the masks the `rng` (REFERENCE) mode applies, drawn on the device.
        kind 0: autoregressive prenet masks uint8 [N,2,256]; kind 1: teacher-forced (keep [B,N,2,256], zone [B,N,4,512])."""
        seed = _rng_seed(rng)
        nk = (1 if kind == 0 else B) * N * 2 * config.PRENET_DIM
        nz = 0 if kind == 0 else B * N * 4 * config.ACOUSTIC_DECODER_DIM
        out = np.empty(nk + nz, np.uint8)
        self._ck(self.lib.vtts_debug_dropout_masks(self.h, int(kind), seed, int(B), int(N), _ptr(out)))
        if kind == 0:
            return out.reshape(N, 2, config.PRENET_DIM)
        return out[:nk].reshape(B, N, 2, config.PRENET_DIM), out[nk:].reshape(B, N, 4, config.ACOUSTIC_DECODER_DIM)

    def acoustic_forward(self, tokens_t, dur_t, N, lengths_t=None, n_frames_t=None, masks_t=None, seed=None, out=None, stream=None,
                         rng=None):
        """vtts_acoustic_forward on torch CUDA tensors, stream-ordered.  Dropout: masks_t, else seed, else rng (the
        reference's own stream drawn on the device), else off."""
        import torch
        assert tokens_t.is_cuda and tokens_t.dtype == torch.int32 and dur_t.dtype == torch.float32
        B, L = tokens_t.shape
        if out is None:
            out = torch.empty((B, N, config.MEL_DIM), dtype=torch.float32, device=tokens_t.device)
        mode = DROPOUT_MASK if masks_t is not None else (DROPOUT_SEED if seed is not None else DROPOUT_OFF)
        if rng is not None:
            mode, seed = DROPOUT_REFERENCE, _rng_seed(rng, masks_t, seed)
        st = torch.cuda.current_stream(tokens_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_acoustic_forward(self.h, _ptr(tokens_t), _ptr(lengths_t), _ptr(dur_t), _ptr(n_frames_t),
                                                _ptr(masks_t), mode, int(seed or 0), B, L, int(N), _ptr(out), st))
        return out

    def duration_forward(self, tokens_t, lengths_t=None, out=None, stream=None):
        import torch
        assert tokens_t.is_cuda and tokens_t.dtype == torch.int32 and tokens_t.is_contiguous()
        B, L = tokens_t.shape
        if out is None:
            out = torch.empty((B, L), dtype=torch.float32, device=tokens_t.device)
        st = torch.cuda.current_stream(tokens_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_duration_forward(self.h, _ptr(tokens_t), _ptr(lengths_t), B, L, _ptr(out), st))
        return out

    def melspec_forward(self, wav_t, out=None, stream=None):
        import torch
        if not self._mel_loaded:
            self.load_mel_filterbank()
        B, S = wav_t.shape
        if out is None:
            out = torch.empty((B, S // config.HOP, config.MEL_DIM), dtype=torch.float32, device=wav_t.device)
        st = torch.cuda.current_stream(wav_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_melspec(self.h, _ptr(wav_t), B, S, _ptr(out), st))
        return out

    # ---- resampling to an output rate (vtts_resample*: scipy.signal.resample_poly with its defaults, fp32) ----
    def resample(self, wav, out_rate: int, in_rate: int = config.SAMPLE_RATE, lengths=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] at `in_rate` -> [ceil(S * up / down)] or [B, that] at `out_rate`, where up /
        down is out_rate / in_rate in lowest terms (each <= 1024).  lengths int [B]: row b holds lengths[b] samples,
        and its outputs past ceil(lengths[b] * up / down) are 0.  Equals scipy.signal.resample_poly(x, up, down) up to
        fp32 rounding; in_rate == out_rate is a copy."""
        x = _np(wav, np.float32)
        one = x.ndim == 1
        x = x[None] if one else x
        if x.ndim != 2 or x.shape[1] < 1:
            raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
        B, S = x.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        y = np.empty((B, resample_length(S, in_rate, out_rate)), np.float32)
        self._ck(self.lib.vtts_resample_host(self.h, _ptr(x), _ptr(lens), B, S, int(in_rate), int(out_rate), _ptr(y)))
        return y[0] if one else y

    def resample_forward(self, x_t, out_rate: int, in_rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, stream=None):
        """vtts_resample on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> [B, ceil(S * up / down)]; lengths_t
        int32 CUDA [B] or None."""
        import torch
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        n = resample_length(S, in_rate, out_rate)
        if out is None:
            out = torch.empty((B, n), dtype=torch.float32, device=x_t.device)
        elif tuple(out.shape) != (B, n) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be contiguous float32 [{B}, {n}]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_resample(self.h, _ptr(x_t), _ptr(lengths_t), B, S, int(in_rate), int(out_rate), _ptr(out), st))
        return out

    def open_resample_stream(self, max_streams: int, max_chunk_samples: int, out_rate: int,
                             in_rate: int = config.SAMPLE_RATE) -> "ResampleStream":
        """Streaming resampler with `max_streams` independent slots (vtts_resample_stream_*): each slot carries its
        filter history across pushes, so its outputs, concatenated, equal `resample` of its whole input bit for bit.
        An output is emitted as soon as every input it reads has arrived (at most `lookahead` samples after its own
        time); END emits the rest."""
        return ResampleStream(self, max_streams, max_chunk_samples, out_rate, in_rate)

    # ---- bias denoiser (vtts_denoise*: STFT spectral subtraction of the vocoder's bias spectrum, fp32) ----
    def denoiser_bias(self, mel=None) -> np.ndarray:
        """The denoiser's bias beta [513]: |X_0|, the magnitude spectrum of frame 0 of the loaded generator's output in
        the current precision mode, for `mel` ([T,80] or [1,T,80]) or by default an all-zero mel [1, 88, 80].  The
        default is computed on first use and kept until the generator or the precision mode changes."""
        import torch
        default = mel is None
        if default and self._denoise_bias is not None:
            return self._denoise_bias.copy()
        m = np.zeros((1, DENOISE_BIAS_FRAMES, config.MEL_DIM), np.float32) if default else _np(mel, np.float32)
        if m.ndim == 2:
            m = m[None]
        if m.ndim != 3 or m.shape[0] != 1 or m.shape[2] != config.MEL_DIM:
            raise ValueError(f"mel must be [T,{config.MEL_DIM}] or [1,T,{config.MEL_DIM}], got {np.shape(mel)}")
        wav = torch.from_numpy(self.mel2wave(m)[0]).to(torch.device("cuda", self.device))
        out = torch.empty(DENOISE_BINS, dtype=torch.float32, device=wav.device)
        st = torch.cuda.current_stream(wav.device).cuda_stream
        self._ck(self.lib.vtts_denoise_bias(self.h, _ptr(wav), int(wav.numel()), _ptr(out), st))
        beta = out.cpu().numpy()
        if default:
            self._denoise_bias = beta.copy()
        return beta

    def _bias_arg(self, bias) -> np.ndarray:
        b = self.denoiser_bias() if bias is None else _np(bias, np.float32, (DENOISE_BINS,), "bias")
        if not (np.all(np.isfinite(b)) and np.all(b >= 0)):
            raise ValueError("bias values must be finite and >= 0")
        return b

    def denoise(self, wav, strength: float, lengths=None, bias=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] -> the same shape with strength * bias subtracted from every STFT magnitude
        (n_fft 1024, hop 256, Hann, reflect-padded centered frames), phase kept; rows of <= 512 samples are copied.
        lengths int [B] in [0, S]: row b holds lengths[b] samples and its outputs past them are 0.  bias f32 [513]
        (default: `denoiser_bias()`)."""
        strength = _strength(strength)
        x = _np(wav, np.float32)
        one = x.ndim == 1
        x = x[None] if one else x
        if x.ndim != 2:
            raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
        B, S = x.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        if S == 0 or B == 0:
            return (x[0] if one else x).copy()          # nothing to transform: empty rows are short rows
        b = self._bias_arg(bias)
        y = np.empty((B, S), np.float32)
        self._ck(self.lib.vtts_denoise_host(self.h, _ptr(x), _ptr(lens), B, S, strength, _ptr(b), _ptr(y)))
        return y[0] if one else y

    def denoise_forward(self, x_t, strength: float, lengths_t=None, bias_t=None, out=None, stream=None):
        """vtts_denoise on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> [B,S]; lengths_t int32 CUDA [B] or None;
        bias_t f32 CUDA [513] or None (`denoiser_bias()`)."""
        import torch
        strength = _strength(strength)
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        if bias_t is None:
            bias_t = torch.from_numpy(self._bias_arg(None)).to(x_t.device)
        elif tuple(bias_t.shape) != (DENOISE_BINS,) or bias_t.dtype != torch.float32 or not bias_t.is_contiguous():
            raise ValueError(f"bias_t must be contiguous float32 [{DENOISE_BINS}]")
        if out is None:
            out = torch.empty((B, S), dtype=torch.float32, device=x_t.device)
        elif tuple(out.shape) != (B, S) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be contiguous float32 [{B}, {S}]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_denoise(self.h, _ptr(x_t), _ptr(lengths_t), B, S, strength, _ptr(bias_t), _ptr(out), st))
        return out

    def open_denoise_stream(self, max_streams: int, max_chunk_samples: int, strength: float, bias=None) -> "DenoiseStream":
        """Streaming denoiser with `max_streams` independent slots (vtts_denoise_stream_*), strength and bias fixed:
        each slot's outputs, concatenated, equal `denoise` of its whole input bit for bit.  An output is emitted once the
        frames covering it are final (at most 1023 samples after its own time); END emits the rest."""
        return DenoiseStream(self, max_streams, max_chunk_samples, strength, bias)

    # ---- pitch shift (vtts_pitch_shift*: a peak-locked phase vocoder on the denoiser's STFT, fp32, double phases) ----
    def pitch_shift(self, wav, semitones, lengths=None) -> np.ndarray:
        """Host arrays: wav f32 [S] or [B,S] -> the same shape, every spectral peak's region moved by the ratio
        fp32(2^(s / 12)) with its phase kept coherent across frames (n_fft 1024, hop 256); the timing of every sample is
        kept.  semitones: a scalar or one value per row, finite and in [-12, 12]; rows with 0 and rows of <= 512 samples
        are copied.  lengths int [B] in [0, S]: row b holds lengths[b] samples and its outputs past them are 0."""
        x = _np(wav, np.float32)
        one = x.ndim == 1
        x = x[None] if one else x
        if x.ndim != 2:
            raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
        B, S = x.shape
        sem = _semitones(semitones, B)
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        if S == 0 or B == 0:
            return (x[0] if one else x).copy()          # nothing to transform: empty rows are short rows
        y = np.empty((B, S), np.float32)
        self._ck(self.lib.vtts_pitch_shift_host(self.h, _ptr(x), _ptr(lens), B, S, _ptr(sem), _ptr(y)))
        return y[0] if one else y

    def pitch_shift_forward(self, x_t, semitones, lengths_t=None, out=None, stream=None):
        """vtts_pitch_shift on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> [B,S] (not x_t); semitones a scalar or
        one host value per row; lengths_t int32 CUDA [B] or None."""
        import torch
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        sem = _semitones(semitones, B)
        if out is None:
            out = torch.empty((B, S), dtype=torch.float32, device=x_t.device)
        elif tuple(out.shape) != (B, S) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be contiguous float32 [{B}, {S}]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_pitch_shift(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(sem), _ptr(out), st))
        return out

    def debug_pitch_decisions(self, x_t, semitones, lengths_t=None) -> np.ndarray:
        """Test hook (vtts_debug_pitch_decisions): int32 [B, S // 256 + 1, 513], the device's peak flags (bit 0) and the
        side of the princarg cut each peak's phase deviation took (bit 1: negative) for `pitch_shift_forward` of the
        same arguments."""
        import torch
        B, S = x_t.shape
        sem = _semitones(semitones, B)
        out = torch.empty((B, S // config.HOP + 1, DENOISE_BINS), dtype=torch.int32, device=x_t.device)
        st = torch.cuda.current_stream(x_t.device).cuda_stream
        self._ck(self.lib.vtts_debug_pitch_decisions(self.h, _ptr(x_t), _ptr(lengths_t), B, S, _ptr(sem), _ptr(out), st))
        return out.cpu().numpy()

    def open_pitch_shift_stream(self, max_streams: int, max_chunk_samples: int) -> "PitchShiftStream":
        """Streaming pitch shifter with `max_streams` independent slots (vtts_pitch_shift_stream_*): a slot's shift is
        given with BEGIN and fixed until END, and its outputs, concatenated, equal `pitch_shift` of its whole input bit
        for bit.  Outputs are released on the denoise stream's schedule (at most 1023 samples after their own time)."""
        return PitchShiftStream(self, max_streams, max_chunk_samples)

    # ---- loudness (vtts_loudness*: ITU-R BS.1770-4 gated loudness and true peak, fp32) ----
    def loudness(self, wav, rate: int = config.SAMPLE_RATE, lengths=None) -> "Loudness":
        """Host arrays: wav f32 [S] or [B,S] at `rate` (a multiple of 10 in [8000, 192000]) -> Loudness of float32 [B]
        arrays (scalars for a 1-D input): integrated, momentary and short-term loudness in LUFS (-inf where undefined) and
        the true peak in dBTP (4x oversampled by resample_poly).  lengths int [B] in [0, S]."""
        rate = _loudness_rate(rate)
        x = _np(wav, np.float32)
        one = x.ndim == 1
        x = x[None] if one else x
        if x.ndim != 2:
            raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
        B, S = x.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        out = np.full((B, 4), -np.inf, np.float32)
        if B and S:                                # empty rows measure as silence
            self._ck(self.lib.vtts_loudness_host(self.h, _ptr(x), _ptr(lens), B, S, rate, _ptr(out)))
        cols = [out[:, i] for i in range(4)]
        return Loudness(*(c[0] for c in cols)) if one else Loudness(*cols)

    def normalize_loudness(self, wav, target: float, rate: int = config.SAMPLE_RATE, true_peak=None, lengths=None):
        """Host arrays: (y, gain_db).  y = wav * fp32(10^(g / 20)) per row with g = target - integrated loudness, at most
        true_peak - the true peak when a ceiling (dBTP, in [-20, 0]) is given; rows measuring -inf are copied (g = 0) and
        outputs past lengths[b] are 0.  target in [-70, 0] LUFS."""
        rate = _loudness_rate(rate)
        target, ceiling = _loudness_target(target, true_peak)
        x = _np(wav, np.float32)
        one = x.ndim == 1
        x = x[None] if one else x
        if x.ndim != 2:
            raise ValueError(f"wav must be [S] or [B,S], got {np.shape(wav)}")
        B, S = x.shape
        lens = None if lengths is None else _np(lengths, np.int32, (B,), "lengths")
        y = x.copy()
        g = np.zeros(B, np.float32)
        if B and S:
            self._ck(self.lib.vtts_loudness_normalize_host(self.h, _ptr(x), _ptr(lens), B, S, rate, target, ceiling, _ptr(y), _ptr(g)))
        return (y[0], g[0]) if one else (y, g)

    def loudness_forward(self, x_t, rate: int = config.SAMPLE_RATE, lengths_t=None, out=None, stream=None):
        """vtts_loudness on torch CUDA tensors, stream-ordered: x_t f32 [B,S] -> f32 [B,4] (integrated, momentary,
        short-term LUFS, true peak dBTP); lengths_t int32 CUDA [B] or None."""
        import torch
        rate = _loudness_rate(rate)
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        if out is None:
            out = torch.empty((B, 4), dtype=torch.float32, device=x_t.device)
        elif tuple(out.shape) != (B, 4) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be contiguous float32 [{B}, 4]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_loudness(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, _ptr(out), st))
        return out

    def normalize_loudness_forward(self, x_t, target: float, rate: int = config.SAMPLE_RATE, true_peak=None, lengths_t=None, out=None,
                                   gain_db=None, stream=None):
        """vtts_loudness_normalize on torch CUDA tensors, stream-ordered and without a host synchronisation: returns
        (y [B,S], gain_db [B]).  `out` may be x_t (in place)."""
        import torch
        rate = _loudness_rate(rate)
        target, ceiling = _loudness_target(target, true_peak)
        assert x_t.is_cuda and x_t.dtype == torch.float32 and x_t.is_contiguous() and x_t.dim() == 2
        B, S = x_t.shape
        if out is None:
            out = torch.empty((B, S), dtype=torch.float32, device=x_t.device)
        elif tuple(out.shape) != (B, S) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be contiguous float32 [{B}, {S}]")
        if gain_db is None:
            gain_db = torch.empty(B, dtype=torch.float32, device=x_t.device)
        elif tuple(gain_db.shape) != (B,) or gain_db.dtype != torch.float32 or not gain_db.is_contiguous():
            raise ValueError(f"gain_db must be contiguous float32 [{B}]")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self._ck(self.lib.vtts_loudness_normalize(self.h, _ptr(x_t), _ptr(lengths_t), B, S, rate, target, ceiling, _ptr(out),
                                                  _ptr(gain_db), st))
        return out, gain_db

    def open_loudness_meter(self, max_streams: int, max_chunk_samples: int, rate: int = config.SAMPLE_RATE,
                            max_seconds: int = 600) -> "LoudnessMeter":
        """Streaming loudness meter with `max_streams` independent slots (vtts_loudness_stream_*): after every push a
        slot's integrated, momentary and short-term readings equal `loudness` of what it has received, bit for bit; its
        true peak lags `lookahead` samples and equals the one-shot value after END.  A slot holds up to `max_seconds`."""
        return LoudnessMeter(self, max_streams, max_chunk_samples, rate, max_seconds)


class Loudness(NamedTuple):
    integrated: np.ndarray     # LUFS (gated, BS.1770-4)
    momentary: np.ndarray      # LUFS, the last 400 ms block
    short_term: np.ndarray     # LUFS, the last 3 s
    true_peak: np.ndarray      # dBTP


def _loudness_rate(rate) -> int:
    r = int(rate)
    if r != rate or r % 10 or not 8000 <= r <= 192000:
        raise ValueError(f"loudness: rate {rate} must be a multiple of 10 in [8000, 192000] (100 ms a whole number of samples)")
    return r


def _loudness_target(target, true_peak):
    """(target, ceiling) as vtts_loudness_normalize takes them: ceiling +inf for none"""
    t = float(target)
    if not -70.0 <= t <= 0.0:
        raise ValueError(f"loudness target {target} LUFS must lie in [-70, 0]")
    if true_peak is None:
        return t, float("inf")
    c = float(true_peak)
    if not (np.isfinite(c) and -20.0 <= c <= 0.0):
        raise ValueError(f"true-peak ceiling {true_peak} dBTP must be finite and lie in [-20, 0]")
    return t, c


STREAM_BEGIN, STREAM_END = 1, 2


class VocoderStream:
    """Handle of a streaming generator (Engine.open_vocoder_stream).  A slot that has received P frames since BEGIN
    has emitted max(0, P - lookahead) frames; a push with END emits the rest."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_frames: int):
        self.eng = eng
        self.max_streams, self.max_chunk_frames = int(max_streams), int(max_chunk_frames)
        self.lookahead = int(eng.lib.vtts_vocoder_stream_lookahead())
        self.wav_ld = config.HOP * (self.max_chunk_frames + self.lookahead)   # samples per slot of the output buffer
        h = C.c_void_p()
        eng._ck(eng.lib.vtts_vocoder_stream_create(eng.h, self.max_streams, self.max_chunk_frames, C.byref(h)))
        self.h = h

    def _host_args(self, n_new, flags):
        S = self.max_streams
        n = _np(n_new, np.int32, (S,), "n_new")
        f = _np(flags, np.uint8, (S,), "flags")
        return n, f

    def push(self, mel, n_new, begin=None, end=None) -> list:
        """mel f32 [S,F',80] (F' <= max_chunk_frames; rows past n_new[s] ignored), n_new int [S], begin / end bool [S]
        or None.  Returns one float32 array per slot with the samples it emits now (256 per frame)."""
        S, F = self.max_streams, self.max_chunk_frames
        mel = _np(mel, np.float32)
        if mel.ndim != 3 or mel.shape[0] != S or mel.shape[1] > F or mel.shape[2] != config.MEL_DIM:
            raise ValueError(f"mel must be [{S}, <= {F}, {config.MEL_DIM}], got {mel.shape}")
        if mel.shape[1] < F:
            mel = np.concatenate([mel, np.zeros((S, F - mel.shape[1], config.MEL_DIM), np.float32)], axis=1)
        flags = np.zeros(S, np.uint8)
        if begin is not None:
            flags |= np.asarray(begin, bool).astype(np.uint8) * STREAM_BEGIN
        if end is not None:
            flags |= np.asarray(end, bool).astype(np.uint8) * STREAM_END
        n, f = self._host_args(n_new, flags)
        wav = np.empty((S, self.wav_ld), np.float32)
        n_out = np.zeros(S, np.int32)
        self.eng._ck(self.eng.lib.vtts_vocoder_stream_push_host(self.eng.h, self.h, _ptr(mel), _ptr(n), _ptr(f), _ptr(wav), _ptr(n_out)))
        return [wav[s, : int(n_out[s]) * config.HOP].copy() for s in range(S)]

    def push_device(self, mel_t, n_new, flags, out_t, stream=None) -> np.ndarray:
        """Device buffers: mel_t f32 CUDA [S,F,80], out_t f32 CUDA [S, 256*(F+lookahead)]; n_new int [S] and flags
        uint8 [S] (bit0 BEGIN, bit1 END) on the host.  Stream-ordered; returns n_out int32 [S] (frames slot s got at
        the start of its row of out_t)."""
        import torch
        S, F = self.max_streams, self.max_chunk_frames
        if tuple(mel_t.shape) != (S, F, config.MEL_DIM) or mel_t.dtype != torch.float32 or not mel_t.is_contiguous():
            raise ValueError(f"mel_t must be contiguous float32 [{S}, {F}, {config.MEL_DIM}]")
        if tuple(out_t.shape) != (S, self.wav_ld) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, {self.wav_ld}]")
        n, f = self._host_args(n_new, flags)
        n_out = np.zeros(S, np.int32)
        st = torch.cuda.current_stream(mel_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_vocoder_stream_push(self.eng.h, self.h, _ptr(mel_t), _ptr(n), _ptr(f), _ptr(out_t), _ptr(n_out), st))
        return n_out

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(self.eng.lib.vtts_vocoder_stream_destroy(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ResampleStream:
    """Handle of a streaming resampler (Engine.open_resample_stream).  Before END a slot that has received P samples
    has emitted min(ceil(P up / down), max(0, floor((P up - 1 - half) / down) + 1)) outputs, half = 10 max(up, down);
    a push with END emits the rest."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, out_rate: int, in_rate: int = config.SAMPLE_RATE):
        self.eng = eng
        self.max_streams, self.max_chunk_samples = int(max_streams), int(max_chunk_samples)
        self.in_rate, self.out_rate = int(in_rate), int(out_rate)
        resample_ratio(self.in_rate, self.out_rate)
        h, pitch = C.c_void_p(), C.c_int()
        eng._ck(eng.lib.vtts_resample_stream_create(eng.h, self.max_streams, self.max_chunk_samples, self.in_rate, self.out_rate,
                                                    C.byref(h), C.byref(pitch)))
        self.h = h
        self.out_pitch = int(pitch.value)   # outputs per slot of a push's output buffer
        self.lookahead = int(eng.lib.vtts_resample_stream_lookahead(self.in_rate, self.out_rate))

    def push(self, x, n_new, begin=None, end=None) -> list:
        """x f32 [S, <= max_chunk_samples] (samples past n_new[s] ignored), n_new int [S], begin / end bool [S] or None.
        Returns one float32 array per slot with the samples it emits now."""
        S, F = self.max_streams, self.max_chunk_samples
        x = _np(x, np.float32)
        if x.ndim != 2 or x.shape[0] != S or x.shape[1] > F:
            raise ValueError(f"x must be [{S}, <= {F}], got {x.shape}")
        if x.shape[1] < F:
            x = np.concatenate([x, np.zeros((S, F - x.shape[1]), np.float32)], axis=1)
        flags = np.zeros(S, np.uint8)
        if begin is not None:
            flags |= np.asarray(begin, bool).astype(np.uint8) * STREAM_BEGIN
        if end is not None:
            flags |= np.asarray(end, bool).astype(np.uint8) * STREAM_END
        n = _np(n_new, np.int32, (S,), "n_new")
        y = np.empty((S, self.out_pitch), np.float32)
        n_out = np.zeros(S, np.int32)
        self.eng._ck(self.eng.lib.vtts_resample_stream_push_host(self.eng.h, self.h, _ptr(x), _ptr(n), _ptr(flags), _ptr(y), _ptr(n_out)))
        return [y[s, : int(n_out[s])].copy() for s in range(S)]

    def push_device(self, x_t, n_new, flags, out_t, stream=None) -> np.ndarray:
        """Device buffers: x_t f32 CUDA [S, max_chunk_samples], out_t f32 CUDA [S, out_pitch]; n_new int [S] and flags
        uint8 [S] (bit0 BEGIN, bit1 END) on the host.  Stream-ordered; returns n_out int32 [S] (outputs slot s got at the
        start of its row of out_t)."""
        import torch
        S, F = self.max_streams, self.max_chunk_samples
        if tuple(x_t.shape) != (S, F) or x_t.dtype != torch.float32 or not x_t.is_contiguous():
            raise ValueError(f"x_t must be contiguous float32 [{S}, {F}]")
        if tuple(out_t.shape) != (S, self.out_pitch) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, {self.out_pitch}]")
        n = _np(n_new, np.int32, (S,), "n_new")
        f = _np(flags, np.uint8, (S,), "flags")
        n_out = np.zeros(S, np.int32)
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_resample_stream_push(self.eng.h, self.h, _ptr(x_t), _ptr(n), _ptr(f), _ptr(out_t), _ptr(n_out), st))
        return n_out

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(self.eng.lib.vtts_resample_stream_destroy(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DenoiseStream:
    """Handle of a streaming denoiser (Engine.open_denoise_stream).  Before END a slot that has received P samples has
    emitted min(P, 256 max(0, floor(P / 256) - 3)) outputs; a push with END emits the rest."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, strength: float, bias=None):
        self.eng = eng
        self.max_streams, self.max_chunk_samples = int(max_streams), int(max_chunk_samples)
        self.strength = _strength(strength)
        self.bias = eng._bias_arg(bias)
        h, pitch = C.c_void_p(), C.c_int()
        eng._ck(eng.lib.vtts_denoise_stream_create(eng.h, self.max_streams, self.max_chunk_samples, self.strength, _ptr(self.bias),
                                                   C.byref(h), C.byref(pitch)))
        self.h = h
        self.out_pitch = int(pitch.value)   # outputs per slot of a push's output buffer
        self.lookahead = int(eng.lib.vtts_denoise_stream_lookahead())

    def push(self, x, n_new, begin=None, end=None) -> list:
        """x f32 [S, <= max_chunk_samples] (samples past n_new[s] ignored), n_new int [S], begin / end bool [S] or None.
        Returns one float32 array per slot with the samples it emits now."""
        S, F = self.max_streams, self.max_chunk_samples
        x = _np(x, np.float32)
        if x.ndim != 2 or x.shape[0] != S or x.shape[1] > F:
            raise ValueError(f"x must be [{S}, <= {F}], got {x.shape}")
        if x.shape[1] < F:
            x = np.concatenate([x, np.zeros((S, F - x.shape[1]), np.float32)], axis=1)
        flags = np.zeros(S, np.uint8)
        if begin is not None:
            flags |= np.asarray(begin, bool).astype(np.uint8) * STREAM_BEGIN
        if end is not None:
            flags |= np.asarray(end, bool).astype(np.uint8) * STREAM_END
        n = _np(n_new, np.int32, (S,), "n_new")
        y = np.empty((S, self.out_pitch), np.float32)
        n_out = np.zeros(S, np.int32)
        self.eng._ck(self.eng.lib.vtts_denoise_stream_push_host(self.eng.h, self.h, _ptr(x), _ptr(n), _ptr(flags), _ptr(y), _ptr(n_out)))
        return [y[s, : int(n_out[s])].copy() for s in range(S)]

    def push_device(self, x_t, n_new, flags, out_t, stream=None) -> np.ndarray:
        """Device buffers: x_t f32 CUDA [S, max_chunk_samples], out_t f32 CUDA [S, out_pitch]; n_new int [S] and flags
        uint8 [S] (bit0 BEGIN, bit1 END) on the host.  Stream-ordered; returns n_out int32 [S] (outputs slot s got at the
        start of its row of out_t)."""
        import torch
        S, F = self.max_streams, self.max_chunk_samples
        if tuple(x_t.shape) != (S, F) or x_t.dtype != torch.float32 or not x_t.is_contiguous():
            raise ValueError(f"x_t must be contiguous float32 [{S}, {F}]")
        if tuple(out_t.shape) != (S, self.out_pitch) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, {self.out_pitch}]")
        n = _np(n_new, np.int32, (S,), "n_new")
        f = _np(flags, np.uint8, (S,), "flags")
        n_out = np.zeros(S, np.int32)
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_denoise_stream_push(self.eng.h, self.h, _ptr(x_t), _ptr(n), _ptr(f), _ptr(out_t), _ptr(n_out), st))
        return n_out

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(self.eng.lib.vtts_denoise_stream_destroy(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PitchShiftStream:
    """Handle of a streaming pitch shifter (Engine.open_pitch_shift_stream).  Before END a slot that has received P samples
    has emitted min(P, 256 max(0, floor(P / 256) - 3)) outputs; a push with END emits the rest."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int):
        self.eng = eng
        self.max_streams, self.max_chunk_samples = int(max_streams), int(max_chunk_samples)
        h, pitch = C.c_void_p(), C.c_int()
        eng._ck(eng.lib.vtts_pitch_shift_stream_create(eng.h, self.max_streams, self.max_chunk_samples, C.byref(h), C.byref(pitch)))
        self.h = h
        self.out_pitch = int(pitch.value)   # outputs per slot of a push's output buffer
        self.lookahead = int(eng.lib.vtts_pitch_shift_stream_lookahead())
        self.shift = np.zeros(self.max_streams, np.float32)   # each slot's shift since its BEGIN

    def _shifts(self, flags, semitones) -> np.ndarray:
        """the semitones array of a push: the given values for the slots that begin, the slots' own shifts elsewhere"""
        sem = self.shift.copy()
        begin = (np.asarray(flags) & STREAM_BEGIN) != 0
        if begin.any():
            if semitones is None:
                raise ValueError("semitones= is required for the slots a push begins")
            given = np.asarray(semitones, np.float32)
            given = np.full(self.max_streams, given, np.float32) if given.ndim == 0 else given
            if given.shape != (self.max_streams,):
                raise ValueError(f"semitones: one value or one per slot ({self.max_streams}), got {np.shape(semitones)}")
            sem[begin] = given[begin]
        return np.ascontiguousarray(sem, np.float32)

    def _commit(self, flags, sem):
        begin = (np.asarray(flags) & STREAM_BEGIN) != 0
        self.shift[begin] = sem[begin]

    def push(self, x, n_new, begin=None, end=None, semitones=None) -> list:
        """x f32 [S, <= max_chunk_samples] (samples past n_new[s] ignored), n_new int [S], begin / end bool [S] or None,
        semitones: a scalar or [S], read for the slots that begin.  Returns one float32 array per slot with the samples
        it emits now."""
        S, F = self.max_streams, self.max_chunk_samples
        x = _np(x, np.float32)
        if x.ndim != 2 or x.shape[0] != S or x.shape[1] > F:
            raise ValueError(f"x must be [{S}, <= {F}], got {x.shape}")
        if x.shape[1] < F:
            x = np.concatenate([x, np.zeros((S, F - x.shape[1]), np.float32)], axis=1)
        flags = np.zeros(S, np.uint8)
        if begin is not None:
            flags |= np.asarray(begin, bool).astype(np.uint8) * STREAM_BEGIN
        if end is not None:
            flags |= np.asarray(end, bool).astype(np.uint8) * STREAM_END
        n = _np(n_new, np.int32, (S,), "n_new")
        sem = self._shifts(flags, semitones)
        y = np.empty((S, self.out_pitch), np.float32)
        n_out = np.zeros(S, np.int32)
        self.eng._ck(self.eng.lib.vtts_pitch_shift_stream_push_host(self.eng.h, self.h, _ptr(x), _ptr(n), _ptr(flags), _ptr(sem), _ptr(y),
                                                                    _ptr(n_out)))
        self._commit(flags, sem)
        return [y[s, : int(n_out[s])].copy() for s in range(S)]

    def push_device(self, x_t, n_new, flags, out_t, semitones=None, stream=None) -> np.ndarray:
        """Device buffers: x_t f32 CUDA [S, max_chunk_samples], out_t f32 CUDA [S, out_pitch]; n_new int [S], flags
        uint8 [S] (bit0 BEGIN, bit1 END) and semitones (scalar or [S], read for the slots that begin) on the host.
        Stream-ordered; returns n_out int32 [S] (outputs slot s got at the start of its row of out_t)."""
        import torch
        S, F = self.max_streams, self.max_chunk_samples
        if tuple(x_t.shape) != (S, F) or x_t.dtype != torch.float32 or not x_t.is_contiguous():
            raise ValueError(f"x_t must be contiguous float32 [{S}, {F}]")
        if tuple(out_t.shape) != (S, self.out_pitch) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, {self.out_pitch}]")
        n = _np(n_new, np.int32, (S,), "n_new")
        f = _np(flags, np.uint8, (S,), "flags")
        sem = self._shifts(f, semitones)
        n_out = np.zeros(S, np.int32)
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_pitch_shift_stream_push(self.eng.h, self.h, _ptr(x_t), _ptr(n), _ptr(f), _ptr(sem), _ptr(out_t),
                                                               _ptr(n_out), st))
        self._commit(f, sem)
        return n_out

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(self.eng.lib.vtts_pitch_shift_stream_destroy(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LoudnessMeter:
    """Handle of a streaming loudness meter (Engine.open_loudness_meter).  Every push returns every slot's readings
    [S,4]: integrated, momentary, short-term LUFS and true peak dBTP of the samples it has received since BEGIN."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_samples: int, rate: int = config.SAMPLE_RATE, max_seconds: int = 600):
        self.eng = eng
        self.max_streams, self.max_chunk_samples = int(max_streams), int(max_chunk_samples)
        self.rate, self.max_seconds = _loudness_rate(rate), int(max_seconds)
        h = C.c_void_p()
        eng._ck(eng.lib.vtts_loudness_stream_create(eng.h, self.max_streams, self.max_chunk_samples, self.rate, self.max_seconds,
                                                    C.byref(h)))
        self.h = h
        self.lookahead = int(eng.lib.vtts_loudness_stream_lookahead(self.rate))

    def push(self, x, n_new, begin=None, end=None) -> np.ndarray:
        """x f32 [S, <= max_chunk_samples] (samples past n_new[s] ignored), n_new int [S], begin / end bool [S] or None.
        Returns float32 [S,4]."""
        S, F = self.max_streams, self.max_chunk_samples
        x = _np(x, np.float32)
        if x.ndim != 2 or x.shape[0] != S or x.shape[1] > F:
            raise ValueError(f"x must be [{S}, <= {F}], got {x.shape}")
        if x.shape[1] < F:
            x = np.concatenate([x, np.zeros((S, F - x.shape[1]), np.float32)], axis=1)
        flags = np.zeros(S, np.uint8)
        if begin is not None:
            flags |= np.asarray(begin, bool).astype(np.uint8) * STREAM_BEGIN
        if end is not None:
            flags |= np.asarray(end, bool).astype(np.uint8) * STREAM_END
        n = _np(n_new, np.int32, (S,), "n_new")
        out = np.empty((S, 4), np.float32)
        self.eng._ck(self.eng.lib.vtts_loudness_stream_push_host(self.eng.h, self.h, _ptr(x), _ptr(n), _ptr(flags), _ptr(out)))
        return out

    def push_device(self, x_t, n_new, flags, out_t, stream=None):
        """Device buffers: x_t f32 CUDA [S, max_chunk_samples], out_t f32 CUDA [S,4]; n_new int [S] and flags uint8 [S]
        (bit0 BEGIN, bit1 END) on the host.  Stream-ordered."""
        import torch
        S, F = self.max_streams, self.max_chunk_samples
        if tuple(x_t.shape) != (S, F) or x_t.dtype != torch.float32 or not x_t.is_contiguous():
            raise ValueError(f"x_t must be contiguous float32 [{S}, {F}]")
        if tuple(out_t.shape) != (S, 4) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, 4]")
        n = _np(n_new, np.int32, (S,), "n_new")
        f = _np(flags, np.uint8, (S,), "flags")
        st = torch.cuda.current_stream(x_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_loudness_stream_push(self.eng.h, self.h, _ptr(x_t), _ptr(n), _ptr(f), _ptr(out_t), st))
        return out_t

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(self.eng.lib.vtts_loudness_stream_destroy(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def acoustic_stream_schedule(n_frames: int, n_emit: int | None, chunk: int, lookahead: int = 10) -> list:
    """Frames an acoustic stream slot emits per push: it scans min(n_frames, n_emit + lookahead) frames, `chunk` per
    push; after P frames scanned it has emitted min(n_emit, max(0, P - lookahead)), and its last push emits the rest."""
    n_emit = n_frames if n_emit is None else n_emit
    end = min(n_frames, n_emit + lookahead)
    P, E, out = 0, 0, []
    while P < end:
        P = min(end, P + chunk)
        e = n_emit if P == end else min(n_emit, max(0, P - lookahead))
        out.append(e - E)
        E = e
    return out


class AcousticStream:
    """Handle of a streaming acoustic model (Engine.open_acoustic_stream)."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int, seed=None, rng=None,
                 masks: bool = False):
        self.eng = eng
        self.max_streams, self.max_chunk_frames = int(max_streams), int(max_chunk_frames)
        self.max_frames, self.max_tokens = int(max_frames), int(max_tokens)
        if rng is not None:
            self.mode, self.seed = DROPOUT_REFERENCE, _rng_seed(rng, seed, True if masks else None)
        elif masks:
            if seed is not None:
                raise ValueError("masks=True selects MASK mode; it cannot be combined with seed=")
            self.mode, self.seed = DROPOUT_MASK, 0
        else:
            self.mode, self.seed = (DROPOUT_SEED if seed is not None else DROPOUT_OFF), int(seed or 0)
        self.lookahead = int(eng.lib.vtts_acoustic_stream_lookahead())
        self.out_frames = self.max_chunk_frames + self.lookahead   # frames per slot of a push's output buffer
        self.open = np.zeros(self.max_streams, bool)               # host mirror of the library's slot state
        self._left = np.zeros(self.max_streams, np.int64)          # pushes left per open slot
        h = C.c_void_p()
        eng._ck(eng.lib.vtts_acoustic_stream_create(eng.h, self.max_streams, self.max_chunk_frames, self.max_frames, self.max_tokens,
                                                    self.mode, self.seed, C.byref(h)))
        self.h = h

    def begin(self, slots, tokens, dur_frames, lengths=None, n_frames=None, n_emit=None, masks=None):
        """Start one utterance per entry of `slots` (closed slots): tokens int [nb,L], durations in frames [nb,L],
        lengths / n_frames as for `predict_mel`, n_emit int [nb] (frames to emit, <= n_frames; default all), masks uint8
        [nb,>=N,2,256] in MASK mode."""
        slots = _np(np.atleast_1d(slots), np.int32)
        if (masks is not None) != (self.mode == DROPOUT_MASK):
            raise ValueError("masks are given to begin exactly when the stream was opened with masks=True")
        tokens, dur, lens, nf, N, masks, _, _ = self.eng._acoustic_args(tokens, dur_frames, lengths, n_frames, masks, None)
        nb, L = tokens.shape
        if slots.shape != (nb,):
            raise ValueError(f"slots must hold one slot per token row ({nb}), got {slots.shape}")
        ne = None if n_emit is None else _np(n_emit, np.int32, (nb,), "n_emit")
        self.eng._ck(self.eng.lib.vtts_acoustic_stream_begin(self.eng.h, self.h, nb, _ptr(slots), _ptr(tokens), _ptr(lens), _ptr(dur),
                                                             _ptr(nf), _ptr(ne), _ptr(masks), L))
        for i, s in enumerate(slots):
            self.open[s] = True
            self._left[s] = len(acoustic_stream_schedule(int(nf[i]), None if ne is None else int(ne[i]), self.max_chunk_frames,
                                                         self.lookahead))

    def _advance(self):
        """slots that close with this push"""
        closing = self.open & (self._left == 1)
        self._left[self.open] -= 1
        self.open &= ~closing
        return closing

    def push(self) -> list:
        """Advance every open slot; returns one float32 [n, 80] array per slot with the frames it emits now."""
        S = self.max_streams
        mel = np.empty((S, self.out_frames, config.MEL_DIM), np.float32)
        n_out = np.zeros(S, np.int32)
        self.eng._ck(self.eng.lib.vtts_acoustic_stream_push_host(self.eng.h, self.h, _ptr(mel), _ptr(n_out)))
        self._advance()
        return [mel[s, : int(n_out[s])].copy() for s in range(S)]

    def push_device(self, out_t, stream=None) -> np.ndarray:
        """Device output: out_t f32 CUDA [S, F + lookahead, 80].  Stream-ordered; returns n_out int32 [S] (frames slot s
        got at the start of its row of out_t)."""
        import torch
        S = self.max_streams
        if tuple(out_t.shape) != (S, self.out_frames, config.MEL_DIM) or out_t.dtype != torch.float32 or not out_t.is_contiguous():
            raise ValueError(f"out_t must be contiguous float32 [{S}, {self.out_frames}, {config.MEL_DIM}]")
        n_out = np.zeros(S, np.int32)
        st = torch.cuda.current_stream(out_t.device).cuda_stream if stream is None else stream
        self.eng._ck(self.eng.lib.vtts_acoustic_stream_push(self.eng.h, self.h, _ptr(out_t), _ptr(n_out), st))
        self._advance()
        return n_out

    def close(self):
        if getattr(self, "h", None) and getattr(self.eng, "h", None):
            self.eng._ck(self.eng.lib.vtts_acoustic_stream_destroy(self.eng.h, self.h))
        self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TtsStream:
    """Handle of a text-to-speech stream (Engine.open_tts_stream): an acoustic stream of max_chunk_frames F feeding a
    vocoder stream of F + the acoustic lookahead frames per push, with a denoise strength a denoise stream after it,
    with semitones a pitch-shift stream, with an output rate a resample stream, and with meter=True a loudness meter of
    the audio `step()` returns last."""

    def __init__(self, eng: Engine, max_streams: int, max_chunk_frames: int, max_frames: int, max_tokens: int, seed=None, rng=None,
                 output_rate=None, denoise=None, meter=False, semitones=None):
        import torch
        if eng.get_precision() == PRECISION_FP32:
            raise ValueError("the tts stream needs the 'bf16x3' or 'fp16' mode (the vocoder stream has no strict fp32 path)")
        if output_rate is not None:
            resample_ratio(config.SAMPLE_RATE, output_rate)
        if denoise is not None:
            denoise = _strength(denoise)
        if meter:
            _loudness_rate(output_rate or config.SAMPLE_RATE)
        if semitones is not None:
            semitones = float(_semitones(semitones, 1)[0])
        self.eng = eng
        self.rs = None
        self.dn = None
        self.ps = None
        self.mt = None
        self.ac = AcousticStream(eng, max_streams, max_chunk_frames, max_frames, max_tokens, seed=seed, rng=rng)
        try:
            self.voc = VocoderStream(eng, max_streams, self.ac.out_frames)
            pitch = self.voc.wav_ld
            if denoise is not None:
                # the vocoder's output buffer is the denoiser's input: n_new = 256 * frames it emitted
                self.dn = DenoiseStream(eng, max_streams, pitch, denoise)
                pitch = self.dn.out_pitch
            if semitones is not None:
                # the previous stage's output buffer is the pitch shifter's input
                self.ps = PitchShiftStream(eng, max_streams, pitch)
                pitch = self.ps.out_pitch
            if output_rate is not None:
                # the previous stage's output buffer is the resampler's input
                self.rs = ResampleStream(eng, max_streams, pitch, output_rate)
                pitch = self.rs.out_pitch
            if meter:
                # the last stage's output buffer is the meter's input; a slot holds at most max_frames of audio
                seconds = -(-int(max_frames) * config.HOP // config.SAMPLE_RATE) + 1
                self.mt = LoudnessMeter(eng, max_streams, pitch, output_rate or config.SAMPLE_RATE, seconds)
        except Exception:
            if getattr(self, "rs", None) is not None:
                self.rs.close()
            if getattr(self, "ps", None) is not None:
                self.ps.close()
            if getattr(self, "dn", None) is not None:
                self.dn.close()
            if getattr(self, "voc", None) is not None:
                self.voc.close()
            self.ac.close()
            raise
        dev = torch.device("cuda", eng.device)
        self._mel = torch.zeros((max_streams, self.ac.out_frames, config.MEL_DIM), dtype=torch.float32, device=dev)
        self._wav = torch.zeros((max_streams, self.voc.wav_ld), dtype=torch.float32, device=dev)
        self._den = None if self.dn is None else torch.zeros((max_streams, self.dn.out_pitch), dtype=torch.float32, device=dev)
        self._psout = None if self.ps is None else torch.zeros((max_streams, self.ps.out_pitch), dtype=torch.float32, device=dev)
        self._semitones = semitones                    # every slot's default shift
        self._shift = np.zeros(max_streams, np.float32)  # the shift of each slot's utterance
        self._out = None if self.rs is None else torch.zeros((max_streams, self.rs.out_pitch), dtype=torch.float32, device=dev)
        self._mout = None if self.mt is None else torch.zeros((max_streams, 4), dtype=torch.float32, device=dev)
        self._mout_h = None if self.mt is None else torch.zeros((max_streams, 4), dtype=torch.float32).pin_memory()
        self._meter = {}
        self._fresh = np.zeros(max_streams, bool)   # begun, no push yet: the next vocoder push carries BEGIN
        self._empty = set()                         # begun with nothing left after the trim: reported empty at the next step

    @property
    def max_streams(self):
        return self.ac.max_streams

    def begin(self, slot: int, tokens, silence_duration=-1.0, semitones=None):
        """Start `tokens` (one row of phoneme ids) in a free slot: durations, the text2mel fix-ups and the trim are
        planned exactly as `Engine.tts` plans them (vtts_tts_plan).  `semitones` overrides the stream's shift for this
        utterance.  Returns the number of frames the slot will vocode."""
        slot = int(slot)
        if self.ac.open[slot] or slot in self._empty:
            raise ValueError(f"slot {slot} is still open")
        if semitones is not None and self.ps is None:
            raise ValueError("the stream was opened without semitones= (no pitch-shift stage)")
        shift = self._semitones if semitones is None else float(_semitones(semitones, 1)[0])
        tok = _np(tokens, np.int32).reshape(1, -1)
        _, frames, nf, ne = self.eng.tts_plan(tok, silence_duration=silence_duration)
        if nf[0] < 1:
            raise ValueError("tts stream: predicted durations sum to less than one frame")
        if ne[0] == 0:
            self._empty.add(slot)
            return 0
        self.ac.begin([slot], tok, frames, n_frames=nf, n_emit=ne)
        self._fresh[slot] = True
        if self.ps is not None:
            self._shift[slot] = shift
        return int(ne[0])

    def busy(self) -> np.ndarray:
        """bool [S]: slots with an utterance still running"""
        b = self.ac.open.copy()
        for s in self._empty:
            b[s] = True
        return b

    def step(self) -> dict:
        """One acoustic push into a device buffer, then one vocoder push of the frames it emitted (BEGIN on a slot's
        first push, END on its last); one synchronisation.  Returns {slot: float32 samples} for every slot that was
        running (possibly empty); a slot whose utterance finished this step is free afterwards."""
        active = self.ac.open.copy()
        closing_before = active.copy()
        n_out = self.ac.push_device(self._mel) if active.any() else np.zeros(self.max_streams, np.int32)
        closed = closing_before & ~self.ac.open
        flags = (self._fresh & active).astype(np.uint8) * STREAM_BEGIN | closed.astype(np.uint8) * STREAM_END
        out = {s: np.zeros(0, np.float32) for s in self._empty}
        self._empty = set()
        if active.any():
            n_wav = self.voc.push_device(self._mel, n_out, flags, self._wav)
            n_wav = n_wav * config.HOP
            src = self._wav
            if self.dn is not None:
                n_wav = self.dn.push_device(src, n_wav, flags, self._den)
                src = self._den
            if self.ps is not None:
                n_wav = self.ps.push_device(src, n_wav, flags, self._psout, semitones=self._shift)
                src = self._psout
            if self.rs is not None:
                n_wav = self.rs.push_device(src, n_wav, flags, self._out)
                src = self._out
            if self.mt is not None:
                self.mt.push_device(src, n_wav, flags, self._mout)
                self._mout_h.copy_(self._mout, non_blocking=True)   # ready once the blocking copy below returns
            wav = src.cpu().numpy()
            for s in np.flatnonzero(active):
                out[int(s)] = wav[s, : int(n_wav[s])].copy()
            if self.mt is not None:
                m = self._mout_h.numpy()
                self._meter = {int(s): tuple(float(v) for v in m[s]) for s in np.flatnonzero(active)}
        self._fresh &= ~active
        return out

    def meter(self) -> dict:
        """{slot: (integrated, momentary, short_term, true_peak)} of the audio each slot stepped last has produced since
        its BEGIN (meter=True): equal to `Engine.loudness` of that audio, bit for bit, once the slot's last step ran."""
        if self.mt is None:
            raise ValueError("the stream was opened without meter=True")
        return dict(self._meter)

    def close(self):
        if getattr(self, "mt", None) is not None:
            self.mt.close()
        if getattr(self, "rs", None) is not None:
            self.rs.close()
        if getattr(self, "ps", None) is not None:
            self.ps.close()
        if getattr(self, "dn", None) is not None:
            self.dn.close()
        if getattr(self, "voc", None) is not None:
            self.voc.close()
        if getattr(self, "ac", None) is not None:
            self.ac.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


_engines: dict = {}
_lock = threading.Lock()


def get_engine(device: int | None = None) -> Engine:
    """Process-wide engine per device (LOCAL_RANK by default under torchrun)."""
    import os
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    with _lock:
        if device not in _engines:
            _engines[device] = Engine(device)
        return _engines[device]
