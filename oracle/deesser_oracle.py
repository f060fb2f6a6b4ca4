"""Float64 statement of the split-band de-esser (vtts_deess*, vtts_deesser_stream_*): the compressor's detector keyed
by the band above a crossover, turning down only that band.

    row x of n samples at rate r (an integer in [8000, 192000]); fp32 parameters freq Hz in [1000, 0.45 r], threshold,
    ratio, knee, attack and release as for the compressor (compressor_oracle.RANGES), range dB in [0, 24]
    1. split: h = sosfilt(sos_hp, x) from zero state, sos_hp the one section of the second-order Butterworth high-pass
       at freq (eq_oracle.butter("high", 2, freq, r), vtts_eq_design(VTTS_EQ_HIGHPASS, r, freq, order=2))
    2. level L = 20 log10 |h|  (-inf where h = 0)
    3. detector: y_L = compressor_oracle.attack(release(reduction(L))) with a = fp32(exp(-1000 / (tau r))), b = 1 - a;
       no makeup
    4. depth cap: y^_L = min(y_L, range), g = 10^(-y^_L / 20)
    5. y = x - (1 - g) h: the low band x - h passes untouched, the high band is scaled by g;  outputs past n are 0
    6. reduction_db = -max_t y^_L  (<= 0)

The device evaluates y as fmaf(g - 1, h, x) where y^_L > 0 and as x where y^_L = 0, so rows whose high band stays below
the knee (and ratio 1, and range 0) come back bit for bit.  The sidechain is the equalizer's filter (1024-sample
blocks) and the detector the compressor's two block scans (256-sample blocks): `yl_by_maps` states the detector in that
form.
"""
from __future__ import annotations

import numpy as np

from oracle import compressor_oracle as co
from oracle import eq_oracle as eo

VOICE = dict(freq=5000.0, threshold=-30.0, ratio=4.0, knee=6.0, attack=1.0, release=60.0, range=12.0)
RANGES = dict(freq=(1000.0, None), threshold=co.RANGES["threshold"], ratio=co.RANGES["ratio"], knee=co.RANGES["knee"],
              attack=co.RANGES["attack"], release=co.RANGES["release"], range=(0.0, 24.0))
DETECTOR = ("threshold", "ratio", "knee", "attack", "release")


def params(rate: int, **kw) -> dict:
    """the fp32 parameters, checked (keys left out take VOICE), with the detector's coefficients"""
    p = {k: co.f32(kw.get(k, v)) for k, v in VOICE.items()}
    if set(kw) - set(VOICE):
        raise ValueError(f"unknown {sorted(set(kw) - set(VOICE))}")
    if not (1000.0 <= p["freq"] <= 0.45 * rate):
        raise ValueError(f"freq {p['freq']}")
    if not (0.0 <= p["range"] <= 24.0):
        raise ValueError(f"range {p['range']}")
    d = co.params(rate, **{k: p[k] for k in DETECTOR})
    return dict(d, freq=p["freq"], range=p["range"])


def highpass(freq: float, rate: int) -> np.ndarray:
    return eo.butter("high", 2, co.f32(freq), rate)


def deess(x, rate: int, parts: bool = False, **kw):
    """(y, reduction_db) of one row in float64; with parts also a dict of h, L, xl, y1, yl, ylc and the parameters"""
    p = params(rate, **kw)
    x = np.asarray(x, np.float32).astype(np.float64)
    h = eo.sosfilt(highpass(p["freq"], rate), x)
    with np.errstate(divide="ignore"):
        L = 20.0 * np.log10(np.abs(h))
    xl = co.reduction(L, p["threshold"], p["ratio"], p["knee"])
    y1 = co.release(xl, p["aR"], p["bR"])
    yl = co.attack(y1, p["aA"], p["bA"])
    ylc = np.minimum(yl, p["range"])
    g = 10.0 ** (-ylc / 20.0)
    y = x - (1.0 - g) * h
    red = -float(ylc.max()) if ylc.size else 0.0
    red = red if red != 0.0 else 0.0
    if parts:
        return y, red, dict(h=h, L=L, xl=xl, y1=y1, yl=yl, ylc=ylc, g=g, **p)
    return y, red


def yl_by_maps(xl, p: dict, t0: int = 0) -> np.ndarray:
    """the capped detector output through the compressor's block maps (sample i of xl is absolute sample t0 + i)"""
    y1 = co.release_by_maps(xl, p["aR"], p["bR"], t0)
    return np.minimum(co.attack_by_maps(y1, p["aA"], p["bA"], t0), p["range"])
