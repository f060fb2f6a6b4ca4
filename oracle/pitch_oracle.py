"""Float64 statement of the pitch shifter (vtts_pitch_shift, vtts_pitch_shift_stream_*): a peak-locked phase vocoder
(Laroche & Dolson, "New phase-vocoder techniques for pitch-shifting, harmonizing and other exotic effects", 1999) on the
bias denoiser's STFT.  The stream releases outputs on the denoiser's schedule, imported from denoise_oracle.

One row x of n samples, a shift of s semitones (finite, in [-12, 12]), r = fp32(2^(s / 12)) computed in double:
    trivial  s == 0 or n <= 512: the row is returned unchanged
    STFT     denoise_oracle.stft: n_fft N = 1024, hop H = 256, periodic Hann, reflect padding 512, F = n // 256 + 1
             frames X_t[k], k = 0..512;  a_t = |X_t|, theta_t = arg X_t
    peaks    a_t[k] > a_t[k-1], a_t[k] >= a_t[k+1], a_t[k] > 0 (neighbours outside [0, 512] count as -1); every bin
             belongs to its nearest peak, the lower one on a tie; a frame without peaks gives Z_t = 0 and psi_t = 0
    phase    omega_t[p] = 2 pi p / N + princarg(theta_t[p] - theta_t-1[p] - 2 pi p H / N) / H  (2 pi p / N at t = 0)
             psi_t(p) = princarg(psi_t-1[p] + H (r - 1) omega_t[p]), psi_t-1[k] the rotation of the peak that owned
             bin k in frame t - 1 (psi_-1 = 0);  princarg(x) = x - 2 pi rint(x / 2 pi)
    remap    D_p = rint((r - 1) p) (half to even); bin k owned by p adds X_t[k] (-1)^D_p e^(i psi_t(p)) to Z_t[k + D_p],
             targets outside [0, 512] dropped, contributions to one target summed in ascending k.  (-1)^D refers the
             phase to the frame centre: without it every change of D's parity inverts the grain.
    ISTFT    the denoiser's: overlap-add of w * irfft(Z_t) over the envelope sum w^2, 512 samples trimmed, length n.
Two choices are discrete, the peak flags and the princarg branch of omega at a peak: which side of the cut the wrapped
deviation e = princarg(theta_t[p] - theta_t-1[p] - 2 pi p H / N) lands on when it is near +-pi (an fp32 spectrum can
also put theta itself on the other side of atan2's cut, which moves d by 2 pi and leaves e alone).  `decisions`
[F, 513] overrides both in the device's encoding (1 | (e < 0) << 1 at a peak, 0 elsewhere; vtts_debug_pitch_decisions):
where the override's side differs from float64's and |e| > pi / 2, e moves by 2 pi to that side.
"""
from __future__ import annotations

import numpy as np

from . import denoise_oracle as do
from .denoise_oracle import (HOP, LOOKAHEAD, N_BINS, N_FFT, PAD, emitted, emitted_closed_form, final_after,  # noqa: F401
                             last_input, lookahead, schedule)

MAX_SEMITONES = 12.0


def ratio(semitones) -> np.float32:
    """r = fp32(2^(s / 12)) of an fp32 shift s, computed in double and rounded once"""
    s = float(np.float32(semitones))
    if not (np.isfinite(s) and -MAX_SEMITONES <= s <= MAX_SEMITONES):
        raise ValueError(f"semitones {semitones} must be finite and lie in [-12, 12]")
    return np.float32(2.0 ** (s / 12.0))


def princarg(x):
    return x - 2.0 * np.pi * np.rint(x / (2.0 * np.pi))


def peak_flags(a) -> np.ndarray:
    """bool [513]: the peaks of one frame's magnitudes"""
    a = np.asarray(a, np.float64)
    ap = np.concatenate([[-1.0], a, [-1.0]])
    return (a > ap[:-2]) & (a >= ap[2:]) & (a > 0)


def owners(flags) -> np.ndarray:
    """int [513]: the nearest peak of every bin, the lower one on a tie; -1 in a frame without peaks"""
    pk = np.flatnonzero(flags)
    k = np.arange(len(flags))
    if pk.size == 0:
        return np.full(k.size, -1)
    li = np.searchsorted(pk, k, side="right") - 1          # last peak <= k
    ri = np.searchsorted(pk, k, side="left")               # first peak >= k
    L = np.where(li >= 0, pk[np.maximum(li, 0)], -1)
    R = np.where(ri < pk.size, pk[np.minimum(ri, pk.size - 1)], -1)
    take_l = (L >= 0) & ((R < 0) | (k - L <= R - k))
    return np.where(take_l, L, R)


def deviation(d, neg=None):
    """e = princarg(d); with `neg` (bool, the side taken) e moves by -+2 pi where it lies on the other side of the cut"""
    e = princarg(d)
    if neg is not None:
        flip = ((e < 0) != neg) & (np.abs(e) > np.pi / 2)
        e = np.where(flip, e - np.sign(e) * 2 * np.pi, e)
    return e


def analysis(x):
    """(X [F, 513] complex, a, theta) of one row (n > 512)"""
    X = do.stft(x)
    return X, np.abs(X), np.angle(X)


def decisions_of(x, semitones) -> np.ndarray:
    """int32 [F, 513]: float64's own decisions in the device's encoding (zeros for a trivial row)"""
    x = np.asarray(x, np.float64)
    F = do.n_frames(x.size)
    dec = np.zeros((F, N_BINS), np.int32)
    if float(np.float32(semitones)) == 0.0 or x.size <= PAD:
        return dec
    _, a, th = analysis(x)
    for t in range(F):
        pk = np.flatnonzero(peak_flags(a[t]))
        neg = np.zeros(pk.size, bool)
        if t > 0:
            neg = deviation(th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * HOP / N_FFT) < 0
        dec[t, pk] = 1 | neg.astype(np.int32) << 1
    return dec


def pitch_shift(x, semitones, decisions=None, frame_centre=True) -> np.ndarray:
    """y of one row in float64 (x taken as float64); `frame_centre=False` drops the (-1)^D factor (a wrong variant)"""
    x = np.asarray(x, np.float64)
    n = x.size
    r = float(ratio(semitones))
    if float(np.float32(semitones)) == 0.0 or n <= PAD:
        return x.copy()
    X, a, th = analysis(x)
    F = X.shape[0]
    k = np.arange(N_BINS)
    Z = np.zeros_like(X)
    psi_prev = np.zeros(N_BINS)
    for t in range(F):
        flags = peak_flags(a[t]) if decisions is None else (np.asarray(decisions[t]) & 1) == 1
        own = owners(flags)
        pk = np.flatnonzero(flags)
        om = 2 * np.pi * pk / N_FFT
        prev = np.zeros(pk.size)
        if t > 0:
            d = th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * HOP / N_FFT
            neg = None if decisions is None else (np.asarray(decisions[t])[pk] >> 1 & 1) == 1
            om = om + deviation(d, neg) / HOP
            prev = psi_prev[pk]
        psi_of = np.zeros(N_BINS)
        psi_of[pk] = princarg(prev + HOP * (r - 1) * om)
        has = own >= 0
        psi_bin = np.where(has, psi_of[np.maximum(own, 0)], 0.0)
        D = np.where(has, np.rint((r - 1) * own), 0).astype(np.int64)
        j = k + D
        ok = has & (j >= 0) & (j < N_BINS)
        sign = np.where(D % 2 == 1, -1.0, 1.0) if frame_centre else np.ones(N_BINS)
        contrib = X[t] * sign * np.exp(1j * psi_bin)
        np.add.at(Z[t], j[ok], contrib[ok])                # unbuffered, in ascending k
        psi_prev = psi_bin
    y_frames = np.fft.irfft(Z, N_FFT, axis=1) * do.window()
    return do.overlap_add(y_frames, n) / do.envelope(n)


def error_scale(x, semitones) -> np.ndarray:
    """per output t: sum over the frames f covering t of w(t_f) ||w x_f||_2 / env(t), the scale of the fp32 rounding
    error (|x| for a trivial row, which is a copy)"""
    x = np.asarray(x, np.float64)
    if float(np.float32(semitones)) == 0.0 or x.size <= PAD:
        return np.abs(x)
    return do.error_scale(x, 0.0, np.zeros(N_BINS))
