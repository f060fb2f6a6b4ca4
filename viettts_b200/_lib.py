"""ctypes binding of libviettts_b200.so (the C ABI in include/viettts_b200.h).

The product path has NO fallback: if the library is missing or cannot be loaded,
importing the binding raises, and every failing call raises VttsError with the
library's message."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libviettts_b200.so"

c_ctx = C.c_void_p
f32p = C.POINTER(C.c_float)
i32p = C.POINTER(C.c_int32)
u8p = C.POINTER(C.c_uint8)
ptrp = C.POINTER(C.c_void_p)   # host array of device pointers

# name -> (restype, argtypes); kept in sync with include/viettts_b200.h by tests/test_abi.py
SIGNATURES = {
    "vtts_version": (C.c_int, []),
    "vtts_create": (C.c_int, [C.c_int, C.POINTER(c_ctx)]),
    "vtts_destroy": (C.c_int, [c_ctx]),
    "vtts_last_error": (C.c_char_p, [c_ctx]),
    "vtts_device_info": (C.c_int, [c_ctx, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]),
    "vtts_set_precision": (C.c_int, [c_ctx, C.c_int]),
    "vtts_get_precision": (C.c_int, [c_ctx]),
    "vtts_debug_conv1d": (C.c_int, [c_ctx, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "vtts_debug_conv_dispatch": (C.c_int, [c_ctx, C.c_int, C.c_int, ptrp, ptrp, ptrp, ptrp, ptrp, ptrp, C.c_void_p,
                                           C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "vtts_debug_tc_stats": (C.c_int, [c_ctx, C.c_int, C.c_void_p]),
    "vtts_debug_substages": (C.c_int, [c_ctx, C.c_int, C.c_void_p]),
    "vtts_debug_dropout_masks": (C.c_int, [c_ctx, C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_void_p]),
    "vtts_debug_pair": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "vtts_debug_pitch_decisions": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_debug_hifigan_layer": (C.c_int, [c_ctx, C.c_int, ptrp, ptrp, C.c_void_p, C.c_int, C.c_int]),
    "vtts_hifigan_blob_floats": (C.c_int64, []),
    "vtts_acoustic_blob_floats": (C.c_int64, []),
    "vtts_duration_blob_floats": (C.c_int64, []),
    "vtts_load_hifigan": (C.c_int, [c_ctx, C.c_void_p, C.c_int64]),
    "vtts_load_duration": (C.c_int, [c_ctx, C.c_void_p, C.c_int64]),
    "vtts_duration_forward": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_predict_duration_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtts_load_acoustic": (C.c_int, [c_ctx, C.c_void_p, C.c_int64]),
    "vtts_load_mel_filterbank": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_int]),
    "vtts_broadcast_weights": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtts_hifigan_forward": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_acoustic_forward": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64,
                                        C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_melspec": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_debug_read": (C.c_int, [c_ctx, C.c_char_p, C.c_void_p, C.c_int64]),
    "vtts_mel2wave_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtts_predict_mel_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64,
                                        C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtts_synthesize_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64,
                                       C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_tts_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_uint64, C.c_int,
                                C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p]),
    "vtts_tts_joined_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_int,
                                       C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p]),
    "vtts_acoustic_teacher_forward": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_gta_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_melspec_host": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtts_vocoder_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "vtts_vocoder_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_vocoder_stream_lookahead": (C.c_int, []),
    "vtts_vocoder_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_vocoder_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_resample_filter": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_int]),
    "vtts_resample": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_resample_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtts_resample_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "vtts_resample_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_resample_stream_lookahead": (C.c_int, [C.c_int, C.c_int]),
    "vtts_resample_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_resample_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_denoise": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_denoise_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]),
    "vtts_denoise_bias": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_denoise_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_float, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "vtts_denoise_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_denoise_stream_lookahead": (C.c_int, []),
    "vtts_denoise_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_denoise_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_pitch_shift": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_pitch_shift_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_pitch_shift_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "vtts_pitch_shift_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_pitch_shift_stream_lookahead": (C.c_int, []),
    "vtts_pitch_shift_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p]),
    "vtts_pitch_shift_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p]),
    "vtts_voice_shift": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_voice_shift_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_voice_shift_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p]),
    "vtts_voice_shift_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p]),
    "vtts_time_stretch_length":(C.c_int64, [C.c_int64, C.c_float]),
    "vtts_time_stretch": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vtts_time_stretch_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]),
    "vtts_debug_time_stretch_decisions": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                    C.c_void_p]),
    "vtts_time_stretch_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "vtts_time_stretch_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_time_stretch_stream_lookahead": (C.c_int, []),
    "vtts_time_stretch_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p]),
    "vtts_time_stretch_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_void_p]),
    "vtts_loudness_filter": (C.c_int, [C.c_int, C.c_void_p]),
    "vtts_loudness": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_loudness_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtts_loudness_normalize": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
    "vtts_loudness_normalize_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                               C.c_void_p, C.c_void_p]),
    "vtts_loudness_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "vtts_loudness_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_loudness_stream_lookahead": (C.c_int, [C.c_int]),
    "vtts_loudness_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_loudness_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_limit": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_limit_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                  C.c_void_p, C.c_void_p]),
    "vtts_loudness_normalize_limited": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                                  C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_loudness_normalize_limited_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                                       C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "vtts_limiter_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_int)]),
    "vtts_limiter_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_limiter_stream_lookahead": (C.c_int, [C.c_int, C.c_float]),
    "vtts_limiter_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p]),
    "vtts_limiter_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p]),
    "vtts_eq_design": (C.c_int, [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_void_p, C.POINTER(C.c_int)]),
    "vtts_eq": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_eq_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "vtts_eq_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "vtts_eq_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_eq_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_eq_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_compress": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_compress_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                     C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "vtts_compressor_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                                C.c_float, C.POINTER(C.c_void_p)]),
    "vtts_compressor_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_compressor_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "vtts_compressor_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]),
    "vtts_deess": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                             C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_deess_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                  C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "vtts_deesser_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                             C.c_float, C.c_float, C.POINTER(C.c_void_p)]),
    "vtts_deesser_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_deesser_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p]),
    "vtts_deesser_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p]),
    "vtts_reverb": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_void_p,
                              C.c_void_p]),
    "vtts_reverb_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_void_p]),
    "vtts_reverb_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_void_p),
                                            C.POINTER(C.c_int)]),
    "vtts_reverb_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_reverb_stream_lookahead": (C.c_int, []),
    "vtts_reverb_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_reverb_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_bed_mix": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                               C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_bed_mix_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                    C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]),
    "vtts_bed_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int, C.c_int,
                                         C.c_longlong, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "vtts_bed_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_bed_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_bed_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "vtts_watermark": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_float, C.c_void_p, C.c_void_p]),
    "vtts_watermark_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_float, C.c_void_p]),
    "vtts_watermark_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_uint64, C.c_float, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "vtts_watermark_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_watermark_stream_lookahead": (C.c_int, []),
    "vtts_watermark_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_watermark_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_watermark_detect": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "vtts_watermark_detect_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p]),
    "vtts_encode": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_encode_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtts_decode": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vtts_decode_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtts_flac_bound": (C.c_int64, [C.c_int, C.c_int]),
    "vtts_flac_encode": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                   C.c_void_p, C.c_void_p]),
    "vtts_flac_encode_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                        C.c_void_p]),
    "vtts_flac_rate_code": (C.c_int, [C.c_int]),
    "vtts_flac_stream_create": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "vtts_flac_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_flac_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_flac_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_acoustic_stream_create":(C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, C.POINTER(C.c_void_p)]),
    "vtts_acoustic_stream_destroy": (C.c_int, [c_ctx, C.c_void_p]),
    "vtts_acoustic_stream_lookahead": (C.c_int, []),
    "vtts_acoustic_stream_begin": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_int]),
    "vtts_acoustic_stream_push": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_acoustic_stream_push_host": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtts_tts_plan": (C.c_int, [c_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    "vtts_launch_count": (C.c_int64, [c_ctx]),
    "vtts_last_stage_ms": (C.c_int, [c_ctx, C.c_int, C.POINTER(C.c_float)]),
}


class VttsError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libviettts_b200 error {code}: {msg}")
        self.code = code


_lib = None


def load() -> C.CDLL:
    """Load the shared library (once).  Raises if it has not been built: there is
    no CPU / PyTorch fallback behind this package."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m viettts_b200.build` "
            "(or __graft_entry__.build()). viettts_b200 has no CPU fallback."
        )
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export the symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(ctx, rc: int) -> None:
    if rc != 0:
        msg = load().vtts_last_error(ctx)
        raise VttsError(rc, msg.decode() if msg else "?")
