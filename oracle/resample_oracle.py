"""Float64 statement of the resampler (vtts_resample, vtts_resample_stream_*): scipy.signal.resample_poly(x, up, down)
with its defaults, written out from the definition, and the emission schedule of the stream.

    (in_rate, out_rate) -> up / down reduced by their gcd;  half = 10 * max(up, down)  (0 when up == down: a copy)
    h[k] = up * w[k] / sum(w),  w[k] = fc * sinc(fc * (k - half)) * kaiser(2 * half + 1, 5)[k],  fc = 1 / max(up, down)
    y[m] = sum over 0 <= i < n with 0 <= m * down + half - i * up <= 2 * half  of  x[i] * h[m * down + half - i * up]
    len(y) = ceil(n * up / down)
"""
from __future__ import annotations

from math import gcd

import numpy as np


def ratio(in_rate: int, out_rate: int):
    """(up, down, half)"""
    g = gcd(int(in_rate), int(out_rate))
    up, down = int(out_rate) // g, int(in_rate) // g
    return up, down, (0 if up == down else 10 * max(up, down))


def design(in_rate: int, out_rate: int) -> np.ndarray:
    """h[0 .. 2 * half] in float64 ([1.0] when up == down)"""
    up, down, half = ratio(in_rate, out_rate)
    if half == 0:
        return np.ones(1)
    fc = 1.0 / max(up, down)
    k = np.arange(2 * half + 1, dtype=np.float64)
    w = fc * np.sinc(fc * (k - half)) * np.kaiser(2 * half + 1, 5.0)
    return up * w / w.sum()


def out_len(n: int, in_rate: int, out_rate: int) -> int:
    up, down, _ = ratio(in_rate, out_rate)
    return -(-int(n) * up // down)


def resample(x, in_rate: int, out_rate: int, h=None, m_range=None) -> np.ndarray:
    """y of one row in float64 (x is taken as float64); `h` overrides the taps (e.g. their fp32 rounding);
    `m_range` = (m0, m1) returns only those outputs"""
    x = np.asarray(x, np.float64)
    up, down, half = ratio(in_rate, out_rate)
    h = design(in_rate, out_rate) if h is None else np.asarray(h, np.float64)
    n = x.size
    m0, m1 = (0, out_len(n, in_rate, out_rate)) if m_range is None else m_range
    m = np.arange(m0, m1, dtype=np.int64)
    j = m * down + half
    top = j // up
    T = -(-(2 * half + 1) // up)
    y = np.zeros(m.size)
    for t in range(T):                       # input top - t, tap j - (top - t) * up
        i = top - t
        k = j - i * up
        ok = (i >= 0) & (i < n) & (k <= 2 * half)
        y[ok] += x[i[ok]] * h[k[ok]]
    return y


def abs_sum(x, in_rate: int, out_rate: int, m_range=None) -> np.ndarray:
    """sum |h * x| per output: the scale of its rounding error"""
    return resample(np.abs(np.asarray(x, np.float64)), in_rate, out_rate, h=np.abs(design(in_rate, out_rate)), m_range=m_range)


def last_input(m, in_rate: int, out_rate: int):
    """index of the last input output m reads (the one with tap index (m * down + half) mod up)"""
    up, down, half = ratio(in_rate, out_rate)
    return (np.asarray(m, np.int64) * down + half) // up


def lookahead(in_rate: int, out_rate: int) -> int:
    """largest floor(last input read - the output's own time m * down / up), over every output"""
    up, down, _ = ratio(in_rate, out_rate)
    m = np.arange(2 * up * down + 1, dtype=np.int64)
    # last_input - m * down / up, floored, in integers: floor((up * last - m * down) / up)
    return int(((up * last_input(m, in_rate, out_rate) - m * down) // up).max())


def emitted(P: int, in_rate: int, out_rate: int, end: bool = False) -> int:
    """outputs a stream slot has emitted after P inputs: every output of the P-sample signal whose last input has
    arrived (all of them after END), by counting"""
    n = out_len(P, in_rate, out_rate)
    if end:
        return n
    return int(np.count_nonzero(last_input(np.arange(n), in_rate, out_rate) < P))


def emitted_closed_form(P: int, in_rate: int, out_rate: int) -> int:
    """the same before END as the library computes it: min(ceil(P up / down), max(0, floor((P up - 1 - half) / down) + 1))"""
    up, down, half = ratio(in_rate, out_rate)
    return min(-(-P * up // down), max(0, (P * up - 1 - half) // down + 1))


def schedule(pushes, in_rate: int, out_rate: int, end_last: bool = True):
    """outputs emitted by each push of a slot, for push sizes `pushes` (END with the last one when end_last)"""
    P, E, out = 0, 0, []
    for q, n in enumerate(pushes):
        P += int(n)
        e = emitted(P, in_rate, out_rate, end=end_last and q == len(pushes) - 1)
        out.append(e - E)
        E = e
    return out
