"""Float64 statement of the voice shifter (vtts_voice_shift, vtts_voice_shift_stream_*): pitch_oracle's pitch shift with
a formant shift phi in semitones (finite, in [-12, 12]) that moves the spectral envelope on its own.

f = fp32(2^(phi / 12)) computed in double, as r is.  phi = None is pitch_oracle.pitch_shift itself.  Otherwise, per
analysis frame t with magnitudes a[k] = |X_t[k]|, k = 0..512:
    m = max_k a[k];  l[k] = ln max(a[k], 1e-4 m, 1e-30)       (a floor 80 dB under the frame's peak)
    c[q] = (l[0] + (-1)^q l[512] + 2 sum_k=1..511 l[k] cos(2 pi k q / 1024)) / 1024, q = 0..Q, Q = 26
                                                             (the real cepstrum of the even extension, rectangular lifter)
    E[k] = c[0] + 2 sum_q=1..Q c[q] cos(2 pi k q / 1024)
Bin k, owned by peak p, lands on t = k + D_p as in the pitch shift and is multiplied after its rotation by
    g = exp(min(E(u) - E[k], ln 10^(24 / 20))),  u = t / f in double,
E(u) linear between E[floor u] and E[min(floor u + 1, 512)], E[512] for u > 512.  The boost is capped at +24 dB, the
attenuation is not.  Rows of <= 512 samples and rows with s == 0 and phi == 0 are copied; a row with s == 0 and phi != 0
runs the vocoder at r = 1, where D_p = 0 and psi = 0, so its output is the STFT filtered by g (it has no decisions).
The lifter order follows order ~ fs / (2 F0max) (Roebel & Rodet, "Efficient spectral envelope estimation and its
application to pitch shifting and envelope preservation", DAFx 2005) with F0max ~ 300 Hz at 16 kHz.
"""
from __future__ import annotations

import numpy as np

from . import denoise_oracle as do
from . import pitch_oracle as po
from .denoise_oracle import HOP, N_BINS, N_FFT, PAD

Q = 26
CAP = np.log(10.0 ** (24.0 / 20.0))
ratio = po.ratio                       # f of phi: the same fp32 rounding of the double power


def cosines() -> np.ndarray:
    """float64 [513, Q + 1]: cos(2 pi k q / 1024)"""
    kq = np.outer(np.arange(N_BINS), np.arange(Q + 1)) % N_FFT
    return np.cos(2.0 * np.pi * kq / N_FFT)


def envelope(a) -> np.ndarray:
    """E [..., 513] of magnitudes a [..., 513]"""
    a = np.asarray(a, np.float64)
    m = a.max(axis=-1, keepdims=True)
    l = np.log(np.maximum(np.maximum(a, 1e-4 * m), 1e-30))
    cs = cosines()
    w = np.full(N_BINS, 2.0)
    w[0] = w[-1] = 1.0
    c = (l * w) @ cs / N_FFT
    v = np.full(Q + 1, 2.0)
    v[0] = 1.0
    return (c * v) @ cs.T


def envelope_at(E, u) -> np.ndarray:
    """E(u): linear between E[floor u] and E[min(floor u + 1, 512)], E[512] for u > 512 (u >= 0)"""
    u = np.asarray(u, np.float64)
    i = np.minimum(np.floor(u), N_BINS - 1).astype(np.int64)
    j = np.minimum(i + 1, N_BINS - 1)
    fr = np.where(u > N_BINS - 1, 0.0, u - i)
    return E[..., i] + fr * (E[..., j] - E[..., i])


def gains(E, k, t, f) -> np.ndarray:
    """g of bins k landing on t under envelope E"""
    return np.exp(np.minimum(envelope_at(E, np.asarray(t, np.float64) / float(f)) - E[k], CAP))


def is_copy(n: int, semitones, formant) -> bool:
    s = float(np.float32(semitones))
    return n <= PAD or (s == 0.0 and (formant is None or float(np.float32(formant)) == 0.0))


def voice_shift(x, semitones, formant=None, decisions=None, force=False, scale=False) -> np.ndarray:
    """y of one row in float64 (x taken as float64).  `force` runs the vocoder on a row the copy rule would copy (a row
    of > 512 samples); `scale=True` returns error_scale's per-frame gain factor instead ([F]: the largest g of the
    frame's bins)"""
    x = np.asarray(x, np.float64)
    n = x.size
    if formant is None and not force:
        return po.pitch_shift(x, semitones, decisions=decisions)
    if is_copy(n, semitones, formant) and not (force and n > PAD):
        return x.copy()
    r = float(po.ratio(semitones))
    f = float(ratio(0.0 if formant is None else formant))
    X, a, th = po.analysis(x)
    F = X.shape[0]
    E = envelope(a) if formant is not None else None
    k = np.arange(N_BINS)
    Z = np.zeros_like(X)
    gain = np.ones(F)
    psi_prev = np.zeros(N_BINS)
    for t in range(F):
        flags = po.peak_flags(a[t]) if decisions is None else (np.asarray(decisions[t]) & 1) == 1
        own = po.owners(flags)
        pk = np.flatnonzero(flags)
        om = 2 * np.pi * pk / N_FFT
        prev = np.zeros(pk.size)
        if t > 0:
            d = th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * HOP / N_FFT
            neg = None if decisions is None else (np.asarray(decisions[t])[pk] >> 1 & 1) == 1
            om = om + po.deviation(d, neg) / HOP
            prev = psi_prev[pk]
        psi_of = np.zeros(N_BINS)
        psi_of[pk] = po.princarg(prev + HOP * (r - 1) * om)
        has = own >= 0
        psi_bin = np.where(has, psi_of[np.maximum(own, 0)], 0.0)
        D = np.where(has, np.rint((r - 1) * own), 0).astype(np.int64)
        j = k + D
        ok = has & (j >= 0) & (j < N_BINS)
        sign = np.where(D % 2 == 1, -1.0, 1.0)
        g = np.ones(N_BINS)
        if E is not None:
            g[ok] = gains(E[t], k[ok], j[ok], f)
            gain[t] = g[ok].max() if ok.any() else 1.0
        contrib = X[t] * sign * np.exp(1j * psi_bin) * g
        np.add.at(Z[t], j[ok], contrib[ok])                # unbuffered, in ascending k
        psi_prev = psi_bin
    if scale:
        return gain
    y_frames = np.fft.irfft(Z, N_FFT, axis=1) * do.window()
    return do.overlap_add(y_frames, n) / do.envelope(n)


def error_scale(x, semitones, formant=None) -> np.ndarray:
    """per output t: sum over the frames f covering t of w(t_f) G_f ||w x_f||_2 / env(t), G_f the largest gain of frame
    f (1 without a formant shift): the pitch shifter's scale with every bin scaled by up to G_f (a weak bin's fp32 phase
    error is carried at its own gain, which can be the frame's largest), |x| for a copied row"""
    x = np.asarray(x, np.float64)
    n = x.size
    if formant is None:
        return po.error_scale(x, semitones)
    if is_copy(n, semitones, formant):
        return np.abs(x)
    w = do.window()
    G = voice_shift(x, semitones, formant, scale=True)
    per_frame = np.linalg.norm(do.frames(x) * w, axis=1) * G
    return do.overlap_add(per_frame[:, None] * w[None, :], n) / do.envelope(n)
