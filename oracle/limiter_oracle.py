"""Float64 statement of the lookahead true-peak limiter (vtts_limit*, vtts_limiter_stream_*) and of loudness
normalization through it.

    row x of n samples at rate r (a multiple of 10 in [8000, 192000]); pre-gain G dB in [-70, 70]; ceiling C dBTP in
    [-20, 0], c = 10^(C / 20); lookahead A ms in [1, 20], W = max(1, rint(A r / 1000)); release R ms in [1, 2000],
    beta = exp(-1000 / (R r))
    1. v = fp32(10^(G / 20)) x
    2. u = resample_poly(v, 4, 1);  p[t] = max(|v[t]|, max |u[j]| over j in [4(t - D), 4(t + D) + 3] inside [0, 4n)),
       D = 10 (the oversampler's half-length in input samples)
    3. tau[t] = min(1, c / p[t]); 1 where p = 0 and past the row's end
    4. hold h[t] = min tau[t .. t + W - 1]
    5. attack a[t] = mean of (1 - h[k]) over k in [t - W + 1, t], h = 1 before sample 0  (so 1 - a[t] <= tau[t])
    6. release in the reduction domain: d[t] = max(a[t], beta d[t - 1] + (1 - beta) a[t]), d[-1] = 0
    7. y[t] = v[t] min(tau[t], 1 - d[t]);  reduction_db = 20 log10(min over t of the applied gain)  (<= 0)

The library realizes step 5 over integers, q = ceil((1 - h) 2^32), rounding the mean up, and step 6 as a scan of the
monotone maps f_t(d) = max(a_t, beta d + e_t), e_t = (1 - beta) a_t, folded in sample order over blocks of Q = 256
samples fixed by absolute index: compositions stay in the closed form M(d) = max(c, m d + k).
"""
from __future__ import annotations

import numpy as np

from . import loudness_oracle as lo

D = lo.LOOKAHEAD             # 10: p[t] reads u over t +- D input samples
OS = lo.OS                   # 4
HALF = OS * D                # 40: resample_poly(x, 4, 1)'s half-length in outputs
Q = 256                      # block of the release scan
MAX_GAIN_DB = 70.0


def params(rate: int, lookahead_ms: float, release_ms: float):
    """(W, beta) in the library's arithmetic: A and R are fp32 values, W = max(1, rint(A r / 1000)) and beta =
    exp(-1000 / (R r)) in double"""
    if not lo.rate_ok(rate):
        raise ValueError(f"rate {rate}")
    A, R = float(np.float32(lookahead_ms)), float(np.float32(release_ms))
    if not (1.0 <= A <= 20.0 and 1.0 <= R <= 2000.0):
        raise ValueError(f"lookahead {A} ms, release {R} ms")
    return max(1, int(np.rint(A * rate / 1000.0))), float(np.exp(-1000.0 / (R * rate)))


def gain_factor(gain_db) -> np.float32:
    """fp32(10^(G / 20)) of the fp32 gain, as gain_apply_kernel rounds it"""
    return np.float32(10.0 ** (float(np.float32(gain_db)) / 20.0))


def peak_env(v) -> np.ndarray:
    """p[t] of step 2"""
    v = np.asarray(v, np.float64)
    n = v.size
    if n == 0:
        return v
    g = np.abs(lo.oversample(v)).reshape(n, OS).max(axis=1)          # max |u| over [4t, 4t + 3]
    gp = np.concatenate([np.zeros(D), g, np.zeros(D)])
    win = np.lib.stride_tricks.sliding_window_view(gp, 2 * D + 1).max(axis=1)
    return np.maximum(np.abs(v), win)


def tau(p, c: float) -> np.ndarray:
    with np.errstate(divide="ignore"):
        return np.where(p > 0, np.minimum(1.0, c / np.where(p > 0, p, 1.0)), 1.0)


def hold(t, W: int) -> np.ndarray:
    tp = np.concatenate([t, np.ones(W - 1)])
    return np.lib.stride_tricks.sliding_window_view(tp, W).min(axis=1)


def attack(h, W: int) -> np.ndarray:
    r = np.concatenate([np.zeros(W - 1), 1.0 - h])
    cs = np.concatenate([[0.0], np.cumsum(r)])
    return (cs[W:] - cs[:-W]) / W


def release(a, beta: float) -> np.ndarray:
    d = np.empty_like(a)
    prev = 0.0
    for i, ai in enumerate(a):
        prev = max(ai, beta * prev + (1.0 - beta) * ai)
        d[i] = prev
    return d


def limit(x, rate: int, ceiling: float, gain_db: float = 0.0, lookahead_ms: float = 5.0, release_ms: float = 100.0,
          parts: bool = False):
    """(y, reduction_db) of one row in float64; with parts also a dict of v, p, tau, h, a, d, g"""
    W, beta = params(rate, lookahead_ms, release_ms)
    c = 10.0 ** (float(np.float32(ceiling)) / 20.0)
    v = float(gain_factor(gain_db)) * np.asarray(x, np.float32).astype(np.float64)
    if v.size == 0:
        out = (v.copy(), 0.0)
        return (*out, {}) if parts else out
    p = peak_env(v)
    t = tau(p, c)
    h = hold(t, W)
    a = attack(h, W)
    d = release(a, beta)
    g = np.minimum(t, 1.0 - d)
    y = v * g
    red = float(20.0 * np.log10(g.min())) if g.min() > 0 else -np.inf
    if parts:
        return y, red, dict(v=v, p=p, tau=t, h=h, a=a, d=d, g=g, W=W, beta=beta, c=c)
    return y, red


# ---- the release scan as maps ----------------------------------------------------------------------------------------
IDENTITY = (-np.inf, 1.0, 0.0)


def fold(M, a_t: float, beta: float, e_t: float, fma=lambda x, y, z: x * y + z):
    """f_t after M = (c, m, k): (max(a_t, fma(beta, c, e_t)), beta m, fma(beta, k, e_t))"""
    c, m, k = M
    return max(a_t, fma(beta, c, e_t)), beta * m, fma(beta, k, e_t)


def apply_map(M, d: float, fma=lambda x, y, z: x * y + z) -> float:
    c, m, k = M
    return max(c, fma(m, d, k))


def release_by_maps(a, beta: float) -> np.ndarray:
    """d[t] through the block scan (float64): per block of Q samples fixed by absolute index, the entering d_in from the
    chain of whole-block maps, then d[t] = (fold of the block up to t)(d_in)"""
    d = np.empty(len(a))
    d_in = 0.0
    for b0 in range(0, len(a), Q):
        M = IDENTITY
        for t in range(b0, min(len(a), b0 + Q)):
            M = fold(M, float(a[t]), beta, (1.0 - beta) * float(a[t]))
            d[t] = apply_map(M, d_in)
        d_in = apply_map(M, d_in)
    return d


# ---- stream schedule -------------------------------------------------------------------------------------------------
def last_input(t: int, W: int) -> int:
    """the last input sample y[t] depends on, by the definition: tau[t + W - 1] (the hold) reads u up to
    4(t + W - 1 + D) + 3, whose last input is floor((j + HALF) / OS)"""
    k = t + W - 1
    j = OS * (k + D) + OS - 1
    return max(k, (j + HALF) // OS)


def released(P: int, W: int, end: bool = False) -> int:
    """outputs a stream slot releases after P inputs, by counting: every t whose last input has arrived"""
    if end:
        return P
    return sum(1 for t in range(P) if last_input(t, W) < P)


def stream_lookahead(W: int) -> int:
    """the closed form the library gives: inputs past sample t that must have arrived before t is released,
    last_input(t) - t = W - 1 + D + floor((OS - 1 + HALF) / OS) = W + D + 9"""
    return W - 1 + D + (OS - 1 + HALF) // OS


# ---- loudness normalization through the limiter ----------------------------------------------------------------------
def normalize_limited(x, rate: int, target: float, ceiling: float, lookahead_ms: float = 5.0, release_ms: float = 100.0):
    """(y, G): measure L, limit x at G = T - L, measure the result L_y, limit x again at G + (T - L_y); G clamped to
    [-70, 70] and left as it is where a reading is -inf"""
    L = lo.measure(x, rate)[0]
    G = float(np.clip(target - L, -MAX_GAIN_DB, MAX_GAIN_DB)) if np.isfinite(L) else 0.0
    y1, _ = limit(x, rate, ceiling, G, lookahead_ms, release_ms)
    Ly = lo.measure(y1, rate)[0]
    if np.isfinite(Ly):
        G = float(np.clip(G + (target - Ly), -MAX_GAIN_DB, MAX_GAIN_DB))
    y, _ = limit(x, rate, ceiling, G, lookahead_ms, release_ms)
    return y, G
