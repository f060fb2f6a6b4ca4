"""Float64 statement of the convolution reverb (vtts_reverb*, vtts_reverb_stream_*) and of its synthetic rooms.

    row x of n samples at rate r (an integer in [8000, 192000]); impulse response h of L taps (1 <= L <= 5 r, finite);
    mix in [0, 1]
    1. c[t] = sum_{i=0}^{min(t, L-1)} h[i] x[t - i]: the causal linear convolution from zero state
    2. y[t] = (1 - mix) x[t] + mix c[t] for t < n; the tail past n is not emitted and outputs past n are 0

c is taken from one float64 FFT of length at least n + L - 1.

Synthetic room (rt60 s, predelay ms, seed): d = round(predelay r / 1000) zeros, then e = default_rng(seed).standard_normal(N),
N = ceil(rt60 r), times 10^(-3 i / (rt60 r)) (60 dB down after rt60), all scaled to unit energy.
"""
from __future__ import annotations

import numpy as np

ROOM = dict(rt60=0.35, predelay=8.0, mix=0.15, seed=0)
HALL = dict(rt60=1.8, predelay=25.0, mix=0.22, seed=0)


def f32(v) -> float:
    return float(np.float32(v))


def convolve(x, h) -> np.ndarray:
    """c[0..n-1] of float64 rows x [n] and h [L]"""
    x = np.asarray(x, np.float64)
    h = np.asarray(h, np.float64)
    n = x.size
    if n == 0:
        return np.zeros(0)
    m = 1 << int(np.ceil(np.log2(max(2, n + h.size - 1))))
    return np.fft.irfft(np.fft.rfft(x, m) * np.fft.rfft(h, m), m)[:n]


def reverb(x, h, mix: float) -> np.ndarray:
    """y of one row in float64 (x and h as float32 values, mix as its float32 value)"""
    x = np.asarray(x, np.float32).astype(np.float64)
    h = np.asarray(h, np.float32).astype(np.float64)
    m = f32(mix)
    return (1.0 - m) * x + m * convolve(x, h)


def synthetic_ir(rt60: float, predelay_ms: float, seed: int, rate: int) -> np.ndarray:
    """the synthetic room's IR in float64 (rt60 and predelay as their float32 values)"""
    rt60, predelay_ms = f32(rt60), f32(predelay_ms)
    d = int(np.round(predelay_ms * rate / 1000.0))
    n = int(np.ceil(rt60 * rate))
    i = np.arange(n)
    h = np.concatenate([np.zeros(d), np.random.default_rng(seed).standard_normal(n) * 10.0 ** (-3.0 * i / (rt60 * rate))])
    return h / np.sqrt(np.sum(h ** 2))


def schroeder_rt60(h, rate: int, lo_db: float = -5.0, hi_db: float = -35.0) -> float:
    """RT60 read off the Schroeder backward integral of h: a least-squares line through its decay between lo_db and
    hi_db, extrapolated to -60 dB"""
    e = np.cumsum(np.asarray(h, np.float64)[::-1] ** 2)[::-1]
    db = 10.0 * np.log10(e / e[0])
    sel = np.flatnonzero((db <= lo_db) & (db >= hi_db))
    slope, _ = np.polyfit(sel / rate, db[sel], 1)
    return -60.0 / slope
