"""Float64 statement of the loudness meter and normalizer (vtts_loudness*, vtts_loudness_stream_*): ITU-R BS.1770-4
gated loudness of one mono row, a 4x-oversampled true peak, the normalization gain and the stream's peak schedule.

    K-weighting: shelf then high-pass biquad from zero state, coefficients as libebur128 derives them for any rate r
    m = r / 10;  E_k = sum of y_t^2 over sub-block k, for the K = floor(n / m) sub-blocks inside the row
    blocks j < J = max(0, K - 3):  z_j = (E_j + E_j+1 + E_j+2 + E_j+3) / 4m,  l_j = -0.691 + 10 log10 z_j
    integrated: A = {j : l_j > -70};  Gamma = -0.691 + 10 log10(mean z over A) - 10;  R = {j in A : l_j > Gamma}
                L = -0.691 + 10 log10(mean z over R),  -inf when A is empty
    momentary l_J-1 (-inf for J = 0);  short-term -0.691 + 10 log10(sum_{k=K-30}^{K-1} E_k / 30m) (-inf for K < 30)
    true peak 20 log10 max(max |x|, max |resample_poly(x, 4, 1)|)  (dBTP; the sample peak is included because the
    Kaiser interpolator reproduces the input samples only to about 2.5e-3)
    gain to a target T with an optional ceiling C: g = T - L, min(g, C - TP); g = 0 when L = -inf
"""
from __future__ import annotations

import numpy as np
from scipy import signal

SHELF_F0, SHELF_G, SHELF_Q, SHELF_VB = 1681.974450955533, 3.999843853973347, 0.7071752369554196, 0.4996667741545416
HP_F0, HP_Q = 38.13547087613982, 0.5003270373253953
ABS_GATE, REL_GATE, OFFSET = -70.0, -10.0, -0.691
OS = 4                       # true-peak oversampling
LOOKAHEAD = 10               # floor(half / up) of resample_poly(x, 4, 1): half = 40

# ITU-R BS.1770-4 Table 1 and 2 (48 kHz)
BS1770_48K = (np.array([1.53512485958697, -2.69169618940638, 1.19839281085285]), np.array([1.0, -1.69065929318241, 0.73248077421585]),
              np.array([1.0, -2.0, 1.0]), np.array([1.0, -1.99004745483398, 0.99007225036621]))


def rate_ok(rate: int) -> bool:
    return 8000 <= rate <= 192000 and rate % 10 == 0


def design(rate: int):
    """(b_shelf, a_shelf, b_hp, a_hp), float64, a[0] = 1"""
    if not rate_ok(rate):
        raise ValueError(f"rate {rate}")
    K = np.tan(np.pi * SHELF_F0 / rate)
    Vh = 10.0 ** (SHELF_G / 20.0)
    Vb = Vh ** SHELF_VB
    a0 = 1.0 + K / SHELF_Q + K * K
    bs = np.array([Vh + Vb * K / SHELF_Q + K * K, 2.0 * (K * K - Vh), Vh - Vb * K / SHELF_Q + K * K]) / a0
    as_ = np.array([1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / SHELF_Q + K * K) / a0])
    K = np.tan(np.pi * HP_F0 / rate)
    a0 = 1.0 + K / HP_Q + K * K
    bh = np.array([1.0, -2.0, 1.0])
    ah = np.array([1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / HP_Q + K * K) / a0])
    return bs, as_, bh, ah


def coeffs10(rate: int) -> np.ndarray:
    """the layout of vtts_loudness_filter: b0 b1 b2 a1 a2 of the shelf, then of the high-pass"""
    bs, as_, bh, ah = design(rate)
    return np.concatenate([bs, as_[1:], bh, ah[1:]])


def kweight(x, rate: int) -> np.ndarray:
    bs, as_, bh, ah = design(rate)
    return signal.lfilter(bh, ah, signal.lfilter(bs, as_, np.asarray(x, np.float64)))


def energies(x, rate: int) -> np.ndarray:
    """E_k of every sub-block wholly inside the row"""
    m = rate // 10
    y = kweight(x, rate)
    K = y.size // m
    return (y[: K * m].reshape(K, m) ** 2).sum(axis=1)


def lufs(z):
    with np.errstate(divide="ignore"):
        return OFFSET + 10.0 * np.log10(z)


def gate(E, m: int):
    """(integrated, momentary, short-term) of sub-block energies E"""
    E = np.asarray(E, np.float64)
    K = E.size
    J = max(0, K - 3)
    z = (E[:J] + E[1:J + 1] + E[2:J + 2] + E[3:J + 3]) / (4 * m)
    l = lufs(z)
    a = l > ABS_GATE
    if not a.any():
        L = -np.inf
    else:
        g = lufs(z[a].mean()) + REL_GATE
        r = a & (l > g)
        L = lufs(z[r].mean())
    mom = l[J - 1] if J else -np.inf
    st = lufs(E[K - 30:].sum() / (30 * m)) if K >= 30 else -np.inf
    return float(L), float(mom), float(st)


def oversample(x) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return signal.resample_poly(x, OS, 1) if x.size else x


def true_peak(x) -> float:
    x = np.asarray(x, np.float64)
    if x.size == 0:
        return -np.inf
    p = max(np.abs(x).max(), np.abs(oversample(x)).max())
    with np.errstate(divide="ignore"):
        return float(20.0 * np.log10(p))


def measure(x, rate: int):
    """(integrated, momentary, short-term, true peak)"""
    return (*gate(energies(x, rate), rate // 10), true_peak(x))


def gain(x, rate: int, target: float, ceiling=None) -> float:
    L, _, _, tp = measure(x, rate)
    if not np.isfinite(L):
        return 0.0
    g = target - L
    return g if ceiling is None else min(g, ceiling - tp)


def peak_covered(P: int, end: bool = False) -> int:
    """oversampled outputs the stream's running peak covers after P samples, by counting: every output of the P-sample
    signal whose last input (floor((u + 40) / 4)) has arrived; all 4P after END"""
    if end:
        return OS * P
    u = np.arange(OS * P, dtype=np.int64)
    return int(np.count_nonzero((u + OS * LOOKAHEAD) // OS < P))


def peak_covered_closed_form(P: int) -> int:
    """the same as the library computes it before END: max(0, 4P - 40)"""
    return max(0, OS * P - OS * LOOKAHEAD)
