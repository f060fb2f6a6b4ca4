"""Float64 statement of the feed-forward compressor (vtts_compress*, vtts_compressor_stream_*): a soft-knee gain
computer on the log level and the smooth decoupled peak detector (Giannoulis, Massberg & Reiss, "Digital Dynamic Range
Compressor Design -- A Tutorial and Analysis", JAES 60(6), 2012, eqs. 4 and 17).

    row x of n samples at rate r (an integer in [8000, 192000]); fp32 parameters threshold T dBFS in [-60, 0], ratio R
    in [1, 20], knee W dB in [0, 24], attack A ms in [0.5, 200], release Rel ms in [5, 5000], makeup M dB in [-24, 24]
    1. level L[t] = 20 log10 |x[t]|  (-inf where x = 0)
    2. gain computer (eq. 4): G(L) = L where 2 (L - T) < -W;  L + (1/R - 1) (L - T + W/2)^2 / (2 W) where
       2 |L - T| <= W;  T + (L - T) / R where 2 (L - T) > W  (W = 0: no middle branch).  x_L = L - G(L) >= 0, exactly 0
       below the knee (also at L = -inf)
    3. release y1[t] = max(x_L[t], a_R y1[t - 1] + b_R x_L[t])
    4. attack y_L[t] = a_A y_L[t - 1] + b_A y1[t]  (both from 0 at t = -1)
       a = fp32(exp(-1000 / (tau r))) in double, b = 1 - a (exact in fp32: a >= 0.78 over the parameter ranges)
    5. y[t] = (x[t] m) 10^(-y_L[t] / 20), m = fp32(10^(M / 20));  reduction_db = -max_t y_L[t]  (<= 0, makeup excluded)

The library scans both stages over blocks of Q = 256 samples fixed by absolute index.  The release steps are the
limiter's monotone maps max(c, m d + k); the attack steps are affine maps m d + k.  Each kind closes under composition,
so a block folds into one map and a row chains the block maps (`release_by_maps`, `attack_by_maps`).
"""
from __future__ import annotations

import numpy as np

Q = 256
VOICE = dict(threshold=-24.0, ratio=3.0, knee=6.0, attack=5.0, release=80.0, makeup=0.0)
RANGES = dict(threshold=(-60.0, 0.0), ratio=(1.0, 20.0), knee=(0.0, 24.0), attack=(0.5, 200.0), release=(5.0, 5000.0),
              makeup=(-24.0, 24.0))


def f32(v) -> float:
    return float(np.float32(v))


def coeff(tau_ms: float, rate: int):
    """(a, b) of a one-pole stage with time constant tau_ms: a = fp32(exp(-1000 / (tau r))), b = 1 - a (exact)"""
    a = np.float32(np.exp(-1000.0 / (f32(tau_ms) * rate)))
    b = np.float32(1.0) - a
    assert float(b) == 1.0 - float(a)
    return float(a), float(b)


def makeup_factor(makeup_db: float) -> float:
    return f32(10.0 ** (f32(makeup_db) / 20.0))


def params(rate: int, threshold=VOICE["threshold"], ratio=VOICE["ratio"], knee=VOICE["knee"], attack=VOICE["attack"],
           release=VOICE["release"], makeup=VOICE["makeup"]) -> dict:
    """the fp32 parameters, checked, with the stage coefficients and the makeup factor"""
    if not (8000 <= rate <= 192000 and rate == int(rate)):
        raise ValueError(f"rate {rate}")
    p = dict(threshold=f32(threshold), ratio=f32(ratio), knee=f32(knee), attack=f32(attack), release=f32(release), makeup=f32(makeup))
    for k, (lo, hi) in RANGES.items():
        if not lo <= p[k] <= hi:
            raise ValueError(f"{k} {p[k]}")
    p["aA"], p["bA"] = coeff(p["attack"], rate)
    p["aR"], p["bR"] = coeff(p["release"], rate)
    p["m"] = makeup_factor(p["makeup"])
    return p


def level(x) -> np.ndarray:
    a = np.abs(np.asarray(x, np.float32).astype(np.float64))
    with np.errstate(divide="ignore"):
        return 20.0 * np.log10(a)


def gain_computer(L, T: float, R: float, W: float) -> np.ndarray:
    """G(L) of eq. 4, literally (finite L)"""
    L = np.asarray(L, np.float64)
    d = 2.0 * (L - T)
    G = np.where(d < -W, L, T + (L - T) / R)
    if W > 0:
        knee = np.abs(d) <= W
        G = np.where(knee, L + (1.0 / R - 1.0) * (L - T + W / 2.0) ** 2 / (2.0 * W), G)
    return G


def reduction(L, T: float, R: float, W: float) -> np.ndarray:
    """x_L = L - G(L) in the form that is exactly 0 below the knee and at L = -inf"""
    L = np.asarray(L, np.float64)
    over = L - T
    s = 1.0 - 1.0 / R
    with np.errstate(invalid="ignore"):
        xl = np.where(2.0 * over > W, s * over, 0.0)
        if W > 0:
            knee = np.abs(2.0 * over) <= W
            xl = np.where(knee, s * (over + W / 2.0) ** 2 / (2.0 * W), xl)
    return np.where(np.isfinite(L), xl, 0.0)


def release(xl, a: float, b: float, y0: float = 0.0) -> np.ndarray:
    y = np.empty(len(xl))
    prev = y0
    for i, v in enumerate(xl):
        prev = max(v, a * prev + b * v)
        y[i] = prev
    return y


def attack(y1, a: float, b: float, y0: float = 0.0) -> np.ndarray:
    y = np.empty(len(y1))
    prev = y0
    for i, v in enumerate(y1):
        prev = a * prev + b * v
        y[i] = prev
    return y


def compress(x, rate: int, parts: bool = False, **kw):
    """(y, reduction_db) of one row in float64; with parts also a dict of L, xl, y1, yl and the parameters"""
    p = params(rate, **kw)
    x = np.asarray(x, np.float32).astype(np.float64)
    L = level(x)
    xl = reduction(L, p["threshold"], p["ratio"], p["knee"])
    y1 = release(xl, p["aR"], p["bR"])
    yl = attack(y1, p["aA"], p["bA"])
    y = (x * p["m"]) * 10.0 ** (-yl / 20.0)
    red = -float(yl.max()) if yl.size else 0.0
    red = red if red != 0.0 else 0.0
    if parts:
        return y, red, dict(L=L, xl=xl, y1=y1, yl=yl, **p)
    return y, red


# ---- the two scans as block maps --------------------------------------------------------------------------------------
IDENTITY = (-np.inf, 1.0, 0.0)


def release_fold(M, v: float, a: float, b: float):
    """max(v, a d + b v) after M = (c, m, k)"""
    c, m, k = M
    e = b * v
    return max(v, a * c + e), a * m, a * k + e


def attack_fold(M, v: float, a: float, b: float):
    """a d + b v after M (c stays -inf)"""
    c, m, k = M
    return c, a * m, a * k + b * v


def apply_map(M, d: float) -> float:
    c, m, k = M
    return max(c, m * d + k)


def _by_maps(v, a, b, fold, t0: int):
    """the stage through the block scan: blocks of Q samples fixed by absolute index (sample i of v is t0 + i), the
    entering value of each from the chain of whole-block maps, then out[t] = (fold of the block up to t)(entering)"""
    out = np.empty(len(v))
    d_in = 0.0
    i = 0
    while i < len(v):
        hi = min(len(v), (t0 + i) // Q * Q + Q - t0)
        M = IDENTITY
        for t in range(i, hi):
            M = fold(M, float(v[t]), a, b)
            out[t] = apply_map(M, d_in)
        d_in = apply_map(M, d_in)
        i = hi
    return out


def release_by_maps(xl, a: float, b: float, t0: int = 0) -> np.ndarray:
    return _by_maps(xl, a, b, release_fold, t0)


def attack_by_maps(y1, a: float, b: float, t0: int = 0) -> np.ndarray:
    return _by_maps(y1, a, b, attack_fold, t0)
