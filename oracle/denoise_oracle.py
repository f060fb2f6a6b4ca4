"""Float64 statement of the bias denoiser (vtts_denoise, vtts_denoise_stream_*): STFT spectral subtraction of the
vocoder's bias spectrum, as the WaveGlow / HiFiGAN `Denoiser` does it, and the emission schedule of the stream.

One row x of n samples, strength s >= 0, bias beta[0..512] >= 0:
    STFT   n_fft 1024, hop 256, periodic Hann w, centered frames with reflect padding of 512 on both sides
           (torch.stft(center=True, pad_mode="reflect")): F = n // 256 + 1 frames, frame f covers samples
           256 f - 512 .. 256 f + 511, X_f[k] for k = 0..512
    gain   |X| = sqrt(re^2 + im^2);  M' = max(|X| - s beta[k], 0);  Y = X M' / |X| where |X| > 0, else 0
    ISTFT  torch.istft(Y, 1024, 256, window=w, center=True, length=n): overlap-add of w * irfft(Y_f), divided by the
           envelope sum_f w^2 of the frames that exist, 512 samples trimmed at the front
    n <= 512 cannot be reflect-padded: the row is returned unchanged.
Default bias: beta = |X_0| of the generator's output for an all-zero mel [1, 88, 80].
"""
from __future__ import annotations

import numpy as np

N_FFT, HOP, PAD = 1024, 256, 512
N_BINS = N_FFT // 2 + 1
ZERO_MEL_FRAMES = 88          # frames of the all-zero mel the default bias is taken from
LOOKAHEAD = 1023              # input samples an output reads past its own time


def window() -> np.ndarray:
    """periodic Hann, float64"""
    k = np.arange(N_FFT, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * k / N_FFT)


def n_frames(n: int) -> int:
    return int(n) // HOP + 1


def frames(x) -> np.ndarray:
    """[F, 1024] unwindowed frames of one row (n > 512)"""
    x = np.asarray(x, np.float64)
    xp = np.pad(x, PAD, mode="reflect")
    idx = HOP * np.arange(n_frames(x.size))[:, None] + np.arange(N_FFT)[None, :]
    return xp[idx]


def stft(x) -> np.ndarray:
    """[F, 513] complex spectra of one row (n > 512)"""
    return np.fft.rfft(frames(x) * window(), axis=1)


def bias_of(wav) -> np.ndarray:
    """beta = |X_0|, the magnitude spectrum of frame 0"""
    return np.abs(stft(wav)[0])


def envelope(n: int) -> np.ndarray:
    """sum of w^2 over the frames covering each output sample of an n-sample row"""
    w2 = window() ** 2
    F = n_frames(n)
    env = np.zeros(N_FFT + HOP * (F - 1))
    for f in range(F):
        env[HOP * f: HOP * f + N_FFT] += w2
    return env[PAD: PAD + n]


def overlap_add(y_frames, n: int) -> np.ndarray:
    """sum of the windowed time frames [F, 1024] at each output sample (not yet divided by the envelope)"""
    F = y_frames.shape[0]
    acc = np.zeros(N_FFT + HOP * (F - 1))
    for f in range(F):
        acc[HOP * f: HOP * f + N_FFT] += y_frames[f]
    return acc[PAD: PAD + n]


def denoise(x, strength: float, bias) -> np.ndarray:
    """y of one row in float64 (x taken as float64)"""
    x = np.asarray(x, np.float64)
    n = x.size
    if n <= PAD:
        return x.copy()
    X = stft(x)
    mag = np.abs(X)
    keep = np.maximum(mag - float(strength) * np.asarray(bias, np.float64)[None, :], 0.0)
    gain = np.divide(keep, mag, out=np.zeros_like(mag), where=mag > 0)
    y_frames = np.fft.irfft(X * gain, N_FFT, axis=1) * window()
    return overlap_add(y_frames, n) / envelope(n)


def error_scale(x, strength: float, bias) -> np.ndarray:
    """per output t: sum over the frames f covering t of w(t_f) (||w x_f||_2 + s ||beta||_2 / 32) / env(t), the scale
    of the fp32 rounding error (||.||_2 / 32 = ||.||_2 / sqrt(1024) turns a spectrum norm into a frame norm)"""
    x = np.asarray(x, np.float64)
    n = x.size
    if n <= PAD:
        return np.abs(x)
    w = window()
    per_frame = np.linalg.norm(frames(x) * w, axis=1) + float(strength) * np.linalg.norm(np.asarray(bias, np.float64)) / 32.0
    return overlap_add(per_frame[:, None] * w[None, :], n) / envelope(n)


# ---- stream schedule ----
def last_input(t):
    """last input sample output t reads: frame floor(t / 256) + 2 ends at 256 floor(t / 256) + 1023"""
    t = np.asarray(t, np.int64)
    return HOP * (t // HOP) + 2 * HOP + PAD - 1


def lookahead() -> int:
    """largest last_input(t) - t over every output"""
    t = np.arange(4 * HOP, dtype=np.int64)
    return int((last_input(t) - t).max())


def final_after(t, P: int):
    """output t is final after P inputs, whatever the row's final length: each frame g covering it (g <= floor(t/256)
    + 2) exists and reads no sample past P - 1, i.e. 256 g + 511 <= P - 1 (which also makes the row longer than 512)"""
    g_last = np.asarray(t, np.int64) // HOP + 2
    return HOP * g_last + PAD - 1 <= P - 1


def emitted(P: int, end: bool = False) -> int:
    """outputs a stream slot has emitted after P inputs, by counting (all P after END)"""
    if end:
        return int(P)
    return int(np.count_nonzero(final_after(np.arange(P), P)))


def emitted_closed_form(P: int) -> int:
    """the same before END as the library computes it: min(P, 256 max(0, floor(P / 256) - 3))"""
    return min(int(P), HOP * max(0, int(P) // HOP - 3))


def schedule(pushes, end_last: bool = True):
    """outputs emitted by each push of a slot, for push sizes `pushes` (END with the last one when end_last)"""
    P, E, out = 0, 0, []
    for q, n in enumerate(pushes):
        P += int(n)
        e = emitted(P, end=end_last and q == len(pushes) - 1)
        out.append(e - E)
        E = e
    return out
