"""Integer statement of the wire encodings (viettts_b200/csrc/encode.cu, vtts_encode / vtts_decode): PCM-16 and G.711
mu-law / A-law of float32 audio, and their expansion back to float32.

Encode, per sample x (float32):
  v = clip(rint(x * 32767), -32768, 32767) with x * 32767 in float64 (exact) and rint rounding half to even; NaN -> 0,
      +-Inf clip (synthesizer.float_to_pcm16 for every non-NaN x);
  pcm16: v as int16;
  ulaw:  G.711 mu-law of the 14-bit p = v >> 2;  alaw: G.711 A-law of the 13-bit p = v >> 3 (arithmetic shifts).
Decode: the G.711 expansion of a code to int16 (mu-law 0x00 -> -32124, the tables of CPython's audioop at width 2), or
the int16 itself for pcm16, then v / 32767 in float32 (the scale synthesizer.read_wav uses).
Outputs past a row's length are the code of 0 (pcm16 0, mu-law 0xFF, A-law 0xD5) when encoding and 0.0 when decoding.

Written out from the G.711 segment rules rather than calling `audioop`, which Python 3.13 removes."""
from __future__ import annotations

import numpy as np

ENCODINGS = ("pcm16", "ulaw", "alaw")
SILENCE = {"pcm16": 0, "ulaw": 0xFF, "alaw": 0xD5}
DTYPES = {"pcm16": np.int16, "ulaw": np.uint8, "alaw": np.uint8}
ULAW_ENDS = np.array([0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF, 0x1FFF], np.int64)
ALAW_ENDS = np.array([0x1F, 0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF], np.int64)


def to_int16(x) -> np.ndarray:
    """int64 v of float32 samples x (any shape)"""
    d = np.asarray(x, np.float32).astype(np.float64) * 32767.0
    v = np.clip(np.rint(np.nan_to_num(d, nan=0.0, posinf=np.inf, neginf=-np.inf)), -32768, 32767)
    return v.astype(np.int64)


def _segment(p, ends) -> np.ndarray:
    """the first index seg with p <= ends[seg] (8 where there is none)"""
    return np.searchsorted(ends, p, side="left").astype(np.int64)


def ulaw_of(v) -> np.ndarray:
    p = np.asarray(v, np.int64) >> 2
    neg = p < 0
    mask = np.where(neg, 0x7F, 0xFF)
    p = np.minimum(np.where(neg, -p, p), 8159) + 33
    seg = _segment(p, ULAW_ENDS)
    code = np.where(seg >= 8, 0x7F, (np.minimum(seg, 7) << 4) | ((p >> (np.minimum(seg, 7) + 1)) & 0xF))
    return (code ^ mask).astype(np.uint8)


def alaw_of(v) -> np.ndarray:
    p = np.asarray(v, np.int64) >> 3
    neg = p < 0
    mask = np.where(neg, 0x55, 0xD5)
    p = np.where(neg, -p - 1, p)
    seg = _segment(p, ALAW_ENDS)
    s7 = np.minimum(seg, 7)
    code = np.where(seg >= 8, 0x7F, (s7 << 4) | (np.where(s7 < 2, p >> 1, p >> s7) & 0xF))
    return (code ^ mask).astype(np.uint8)


def ulaw_to_int16(c) -> np.ndarray:
    u = ~np.asarray(c, np.int64) & 0xFF
    t = (((u & 0xF) << 3) + 0x84) << ((u & 0x70) >> 4)
    return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)


def alaw_to_int16(c) -> np.ndarray:
    a = np.asarray(c, np.int64) ^ 0x55
    seg = (a & 0x70) >> 4
    t = ((a & 0xF) << 4) + np.where(seg == 0, 8, 0x108)
    t = t << np.maximum(seg - 1, 0)
    return np.where(a & 0x80, t, -t).astype(np.int16)


def encode(x, encoding: str, lengths=None) -> np.ndarray:
    """codes of float32 x [S] or [B,S] (int16 for pcm16, uint8 for the G.711 laws); past lengths[b] the code of 0"""
    v = to_int16(x)
    y = {"pcm16": lambda: v.astype(np.int16), "ulaw": lambda: ulaw_of(v), "alaw": lambda: alaw_of(v)}[encoding]()
    if lengths is not None:
        y = np.atleast_2d(y).copy()
        for b, n in enumerate(lengths):
            y[b, max(int(n), 0):] = SILENCE[encoding]
        y = y.reshape(np.shape(v))
    return y


def decode_int16(c, encoding: str) -> np.ndarray:
    if encoding == "pcm16":
        return np.asarray(c, np.int16)
    return ulaw_to_int16(c) if encoding == "ulaw" else alaw_to_int16(c)


def decode(c, encoding: str, lengths=None) -> np.ndarray:
    """float32 samples of codes c [S] or [B,S]; 0 past lengths[b]"""
    y = decode_int16(c, encoding).astype(np.float32) / np.float32(32767.0)
    if lengths is not None:
        y = np.atleast_2d(y).copy()
        for b, n in enumerate(lengths):
            y[b, max(int(n), 0):] = 0.0
        y = y.reshape(np.shape(c))
    return y
