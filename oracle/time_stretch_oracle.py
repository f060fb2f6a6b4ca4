"""Float64 statement of the time stretcher (vtts_time_stretch, vtts_time_stretch_stream_*) and of the one phase-vocoder
routine it shares with the pitch shifter (Laroche & Dolson, "Improved phase vocoder time-scale modification of audio",
IEEE TSAP 7(3), 1999; the peaks, owners and princarg of pitch_oracle).  `pitch_shift` here is pitch_oracle.pitch_shift
stated as one case of `vocode`, and reproduces it bit for bit.

One routine, `vocode`, takes a row x of n > 512 samples, a ratio r and the centres a_t of its analysis frames:
    STFT     n_fft N = 1024, periodic Hann, frame t reads samples a_t - 512 .. a_t + 511 reflected at 0 and n - 1;
             X_t[k], k = 0..512;  mag_t = |X_t|, theta_t = arg X_t;  h_t = a_t - a_t-1, h_0 = H = 256 (h_t >= 1)
    peaks    as pitch_oracle: mag_t[k] > mag_t[k-1], mag_t[k] >= mag_t[k+1], mag_t[k] > 0; nearest peak, lower on a tie
    phase    omega_t[p] = 2 pi p / N + princarg(theta_t[p] - theta_t-1[p] - 2 pi p h_t / N) / h_t  (2 pi p / N at t = 0)
             psi_t(p) = princarg(psi_t-1[p] + (H r - h_t) omega_t[p]), psi_t-1[k] the rotation of the peak that owned
             bin k in frame t - 1 (psi_-1 = 0)
    remap    D_p = rint((r - 1) p); bin k owned by p adds X_t[k] (-1)^D_p e^(i psi_t(p)) to Z_t[k + D_p] (ascending k)
    ISTFT    the denoiser's: overlap-add of w * irfft(Z_t) at hop H over the envelope sum w^2, 512 samples trimmed.

Pitch shift by s semitones: r = fp32(2^(s / 12)), a_t = 256 t for F = n // 256 + 1 frames, n outputs ((H r - 256)
equals H (r - 1) exactly in double).  s == 0 or n <= 512: a copy.
Time stretch at tempo alpha (fp32, finite, in [0.5, 2], > 1 faster): M = floor(n / (double)alpha + 0.5) outputs,
T = M // 256 + 1 frames, a_t = min(rint(256 t (double)alpha), n - 1), r = 1 (so D_p = 0 and psi_0 = 0).  alpha == 1 or
n <= 512: the first min(n, M) samples, then zeros up to M.

The discrete decisions (peak flags, princarg side) and their override `decisions` are pitch_oracle's, in the encoding of
vtts_debug_time_stretch_decisions.  The stream schedule is stated at the end.
"""
from __future__ import annotations

import numpy as np

from . import denoise_oracle as do
from .denoise_oracle import HOP, N_BINS, N_FFT, PAD
from .pitch_oracle import deviation, owners, peak_flags, princarg, ratio  # noqa: F401

MIN_TEMPO, MAX_TEMPO = 0.5, 2.0
TS_LOOKAHEAD = 1536           # before END a time-stretch slot has released more than P / alpha - 1536 outputs


def tempo_of(tempo) -> float:
    """the fp32 tempo as a double, checked to be finite and in [0.5, 2]"""
    a = float(np.float32(tempo))
    if not (np.isfinite(a) and MIN_TEMPO <= a <= MAX_TEMPO):
        raise ValueError(f"tempo {tempo} must be finite and lie in [0.5, 2]")
    return a


def stretch_length(n: int, tempo) -> int:
    """M = floor(n / (double)alpha + 0.5)"""
    return int(np.floor(int(n) / tempo_of(tempo) + 0.5))


def stretch_centres(n: int, tempo) -> np.ndarray:
    """int64 [T]: a_t = min(rint(256 t (double)alpha), n - 1) of the T = M // 256 + 1 analysis frames"""
    t = np.arange(do.n_frames(stretch_length(n, tempo)), dtype=np.int64)
    return np.minimum(np.rint(256.0 * t * tempo_of(tempo)).astype(np.int64), int(n) - 1)


def frames_at(x, a) -> np.ndarray:
    """[len(a), 1024] unwindowed frames of one row (n > 512) centred at a, reflected at 0 and n - 1"""
    xp = np.pad(np.asarray(x, np.float64), PAD, mode="reflect")
    return xp[np.asarray(a, np.int64)[:, None] + np.arange(N_FFT)[None, :]]


def hops(a) -> np.ndarray:
    """h_t = a_t - a_t-1 with h_0 = H; every h_t >= 1"""
    a = np.asarray(a, np.int64)
    h = np.diff(a, prepend=a[0] - HOP)
    assert np.all(h >= 1), h.min()
    return h


def analysis(x, a=None):
    """(X [frames, 513] complex, magnitude, theta) of one row (n > 512), frames at a (default 256 t, the STFT's)"""
    X = do.stft(x) if a is None else np.fft.rfft(frames_at(x, a) * do.window(), axis=1)
    return X, np.abs(X), np.angle(X)


def _decisions(x, a) -> np.ndarray:
    _, mag, th = analysis(x, a)
    h = hops(a)
    dec = np.zeros((len(a), N_BINS), np.int32)
    for t in range(len(a)):
        pk = np.flatnonzero(peak_flags(mag[t]))
        neg = np.zeros(pk.size, bool)
        if t > 0:
            neg = deviation(th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * h[t] / N_FFT) < 0
        dec[t, pk] = 1 | neg.astype(np.int32) << 1
    return dec


def decisions_of(x, semitones) -> np.ndarray:
    """pitch_oracle.decisions_of restated through `_decisions`: float64's own decisions of the pitch shifter"""
    x = np.asarray(x, np.float64)
    F = do.n_frames(x.size)
    if float(np.float32(semitones)) == 0.0 or x.size <= PAD:
        return np.zeros((F, N_BINS), np.int32)
    return _decisions(x, HOP * np.arange(F))


def stretch_decisions_of(x, tempo) -> np.ndarray:
    """int32 [T, 513]: float64's own decisions of the time stretcher in the device's encoding (zeros for a trivial row)"""
    x = np.asarray(x, np.float64)
    if tempo_of(tempo) == 1.0 or x.size <= PAD:
        return np.zeros((do.n_frames(stretch_length(x.size, tempo)), N_BINS), np.int32)
    return _decisions(x, stretch_centres(x.size, tempo))


def vocode(x, r: float, a, decisions=None, frame_centre=True) -> np.ndarray:
    """Z [len(a), 513]: the synthesized spectra of one row (n > 512) at ratio r with analysis frames centred at a"""
    X, mag, th = analysis(x, a)
    h = hops(a)
    k = np.arange(N_BINS)
    Z = np.zeros_like(X)
    psi_prev = np.zeros(N_BINS)
    for t in range(X.shape[0]):
        flags = peak_flags(mag[t]) if decisions is None else (np.asarray(decisions[t]) & 1) == 1
        own = owners(flags)
        pk = np.flatnonzero(flags)
        om = 2 * np.pi * pk / N_FFT
        prev = np.zeros(pk.size)
        if t > 0:
            d = th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * h[t] / N_FFT
            neg = None if decisions is None else (np.asarray(decisions[t])[pk] >> 1 & 1) == 1
            om = om + deviation(d, neg) / h[t]
            prev = psi_prev[pk]
        psi_of = np.zeros(N_BINS)
        psi_of[pk] = princarg(prev + (HOP * r - h[t]) * om)
        has = own >= 0
        psi_bin = np.where(has, psi_of[np.maximum(own, 0)], 0.0)
        D = np.where(has, np.rint((r - 1) * own), 0).astype(np.int64)
        j = k + D
        ok = has & (j >= 0) & (j < N_BINS)
        sign = np.where(D % 2 == 1, -1.0, 1.0) if frame_centre else np.ones(N_BINS)
        contrib = X[t] * sign * np.exp(1j * psi_bin)
        np.add.at(Z[t], j[ok], contrib[ok])                # unbuffered, in ascending k
        psi_prev = psi_bin
    return Z


def synthesize(Z, m: int) -> np.ndarray:
    """the denoiser's inverse and overlap-add of Z [m // 256 + 1, 513] into m outputs"""
    y_frames = np.fft.irfft(Z, N_FFT, axis=1) * do.window()
    return do.overlap_add(y_frames, m) / do.envelope(m)


def pitch_shift(x, semitones, decisions=None, frame_centre=True) -> np.ndarray:
    """pitch_oracle.pitch_shift restated as the tempo-1 case of `vocode` (analysis at 256 t, ratio r); the two agree
    bit for bit"""
    x = np.asarray(x, np.float64)
    n = x.size
    r = float(ratio(semitones))
    if float(np.float32(semitones)) == 0.0 or n <= PAD:
        return x.copy()
    return synthesize(vocode(x, r, HOP * np.arange(do.n_frames(n)), decisions, frame_centre), n)


def time_stretch(x, tempo, decisions=None) -> np.ndarray:
    """y of one row in float64 (x taken as float64), M = stretch_length(n, tempo) samples"""
    x = np.asarray(x, np.float64)
    n, M = x.size, stretch_length(x.size, tempo)
    if tempo_of(tempo) == 1.0 or n <= PAD:
        y = np.zeros(M)
        y[: min(n, M)] = x[: min(n, M)]
        return y
    return synthesize(vocode(x, 1.0, stretch_centres(n, tempo), decisions), M)


def stretch_error_scale(x, tempo) -> np.ndarray:
    """error_scale of the time stretcher: per output u, the sum over the synthesis frames f covering u of
    w(u_f) ||w x_f||_2 / env(u), x_f the analysis frame f (|y| for a trivial row, which is a copy)"""
    x = np.asarray(x, np.float64)
    if tempo_of(tempo) == 1.0 or x.size <= PAD:
        return np.abs(time_stretch(x, tempo))
    w = do.window()
    M = stretch_length(x.size, tempo)
    per_frame = np.linalg.norm(frames_at(x, stretch_centres(x.size, tempo)) * w, axis=1)
    return do.overlap_add(per_frame[:, None] * w[None, :], M) / do.envelope(M)


# ---- time-stretch stream schedule ----
def stretch_scanned(P: int, tempo) -> int:
    """frames a slot has scanned before END after P inputs: those with a_t + 512 <= P (unclamped), once P > 512"""
    if P <= PAD:
        return 0
    a = tempo_of(tempo)
    lo, hi = 0, int(P)                  # a_q >= 128 q, so q = P is never scanned; bisect the monotone a_q
    while lo < hi:
        q = (lo + hi) // 2
        if int(np.rint(256.0 * q * a)) + PAD <= P:
            lo = q + 1
        else:
            hi = q
    return lo


def stretch_emitted(P: int, tempo, end: bool = False) -> int:
    """outputs a time-stretch slot has released after P inputs: M at END, P at tempo 1, else max(0, 256 Q - 511) after
    Q scanned frames: output u is weighed by the synthesis frames g with 256 g < u + 512 <= 256 g + 1023 (sample 0 of a
    frame has weight w[0] = 0), all of them scanned"""
    if end:
        return stretch_length(P, tempo)
    if tempo_of(tempo) == 1.0:
        return int(P)
    return max(0, HOP * stretch_scanned(P, tempo) - (PAD - 1))


def stretch_schedule(pushes, tempo, end_last: bool = True):
    """outputs a time-stretch slot releases per push, for push sizes `pushes` (END with the last one when end_last)"""
    P, E, out = 0, 0, []
    for q, n in enumerate(pushes):
        P += int(n)
        e = stretch_emitted(P, tempo, end=end_last and q == len(pushes) - 1)
        out.append(e - E)
        E = e
    return out
