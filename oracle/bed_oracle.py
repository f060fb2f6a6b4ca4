"""Float64 statement of the voice-keyed background bed (vtts_bed_mix*, vtts_bed_stream_*): a looped music or ambience
bed under the speech, turned down by the compressor's detector while the voice is present.

    speech row x of n samples at rate r (an integer in [8000, 192000]); a bed b of Nb samples already at r and already
    at its level; fp32 parameters duck D dB in [0, 40], threshold T dBFS in [-60, 0], attack ms in [0.5, 200], release
    ms in [5, 5000]; sample counts Fi (fade-in), Tt (tail), C (crossfade, 2 C < Nb) and o (start offset, o < Nb)
    1. key level L[t] = 20 log10 |x[t]|, x[t] = 0 for t >= n;  y_L = compressor_oracle's gain computer, release and
       attack with ratio 20 and knee 6 dB
    2. duck: y^_L = min(y_L, D);  g = 10^(-y^_L / 20)
    3. looped bed, P = Nb - C, u = (t + o) mod P:  bl[t] = b[u] for u >= C, else sin(pi u / 2C) b[u] + cos(pi u / 2C)
       b[P + u] (the equal-power crossfade of the bed's end into its start)
    4. envelopes: e_in[t] = (1 - cos(pi t / Fi)) / 2 for t < Fi, else 1;  e_out[t] = (1 + cos(pi (t - n + 1) / Tt)) / 2
       for t >= n, else 1 (the last tail sample is 0);  e = e_in e_out
    5. y[t] = x[t] + g[t] e[t] bl[t] for t < n + Tt;  reduction_db = -max_t y^_L  (<= 0)
    6. a row without a bed returns x and has no tail (reduction 0)

The device evaluates y as fmaf(g e, bl, x) with the compressor's two block scans (256-sample blocks fixed by absolute
index) over the key row x followed by Tt zeros.
"""
from __future__ import annotations

import numpy as np

from oracle import compressor_oracle as co

RATIO, KNEE = 20.0, 6.0
DEFAULTS = dict(duck=12.0, threshold=-40.0, attack=10.0, release=500.0)


def params(rate: int, duck=DEFAULTS["duck"], threshold=DEFAULTS["threshold"], attack=DEFAULTS["attack"],
           release=DEFAULTS["release"]) -> dict:
    """the fp32 parameters, checked, with the detector's coefficients"""
    d = co.params(rate, threshold=threshold, ratio=RATIO, knee=KNEE, attack=attack, release=release)
    D = co.f32(duck)
    if not 0.0 <= D <= 40.0:
        raise ValueError(f"duck {D}")
    return dict(d, duck=D)


def looped(b, T: int, C: int, o: int, weight: bool = False):
    """bl[t], t < T: the bed looped with period P = Nb - C from offset o, the seam crossfaded over u < C; with weight
    also |b[u]| (+ |b[P + u]| over the crossfade), what the crossfade's weights multiply"""
    b = np.asarray(b, np.float32).astype(np.float64)
    P = b.size - C
    assert C >= 0 and 2 * C < b.size and 0 <= o
    u = (np.arange(T) + o) % P
    bl = b[u]
    bw = np.abs(bl)
    if C > 0:
        m = u < C
        w = u[m] / (2.0 * C)
        bl[m] = np.sin(np.pi * w) * b[u[m]] + np.cos(np.pi * w) * b[P + u[m]]
        bw[m] += np.abs(b[P + u[m]])
    return (bl, bw) if weight else bl


def envelope(n: int, Fi: int, Tt: int) -> np.ndarray:
    """e[t], t < n + Tt: the raised-cosine fade-in over [0, Fi) times the raised-cosine fade-out over [n, n + Tt)"""
    t = np.arange(n + Tt, dtype=np.float64)
    e = np.ones(n + Tt)
    if Fi > 0:
        m = t < Fi
        e[m] = 0.5 - 0.5 * np.cos(np.pi * t[m] / Fi)
    if Tt > 0:
        e[n:] *= 0.5 + 0.5 * np.cos(np.pi * (t[n:] - n + 1) / Tt)
    return e


def mix(x, b, rate: int, Fi: int = 0, Tt: int = 0, C: int = 0, o: int = 0, parts: bool = False, **kw):
    """(y [n + Tt], reduction_db) of one row in float64 over the bed b (None: no bed, y = x); with parts also a dict of
    L, xl, y1, yl, ylc, g, e, bl, bw (see `looped`), key and the parameters"""
    p = params(rate, **kw)
    x = np.asarray(x, np.float32).astype(np.float64)
    if b is None:
        return (x.copy(), 0.0, dict(p)) if parts else (x.copy(), 0.0)
    n = x.size
    key = np.concatenate([x, np.zeros(Tt)])
    L = co.level(key)
    xl = co.reduction(L, p["threshold"], p["ratio"], p["knee"])
    y1 = co.release(xl, p["aR"], p["bR"])
    yl = co.attack(y1, p["aA"], p["bA"])
    ylc = np.minimum(yl, p["duck"])
    g = 10.0 ** (-ylc / 20.0)
    e = envelope(n, Fi, Tt)
    bl, bw = looped(b, n + Tt, C, o, weight=True)
    y = key + g * e * bl
    red = -float(ylc.max()) if ylc.size else 0.0
    red = red if red != 0.0 else 0.0
    if parts:
        return y, red, dict(L=L, xl=xl, y1=y1, yl=yl, ylc=ylc, g=g, e=e, bl=bl, bw=bw, key=key, **p)
    return y, red
