"""CPU restatement of MelFilter (STFT + log-mel).  Test infrastructure only.

Pinned to the output of the reference's own dsp.py executed on numpy stand-ins for jax / librosa
(tests/refshim, tests/golden/nat_ref_gta.npz `logmel`, tests/test_reference_goldens.py).
Follows the reference's vietTTS/nat/dsp.py:

  rolling_window   dsp.py:11-25
  batched_stft     dsp.py:65-101  (center=False path; periodic Hann = hanning(1025)[:-1])
  MelFilter        dsp.py:104-128

librosa.filters.mel (un-vendored dependency, setup.py:13) is restated from its
published algorithm (Slaney mel scale, Slaney area normalisation) in
`librosa_mel_filterbank` and cross-checked in tests against torchaudio's
independent implementation.
"""
from __future__ import annotations

import numpy as np


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, mels)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), freqs)


def librosa_mel_filterbank(sr=16000, n_fft=1024, n_mels=80, fmin=0.0, fmax=8000.0) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) -> float32 [n_mels, 1+n_fft//2]
    (htk=False, norm='slaney'), as called at dsp.py:109-111."""
    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, float(sr) / 2, n_bins, endpoint=True)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, n_bins), dtype=np.float64)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2 : n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, None]
    return weights.astype(np.float32)


def rolling_window(a: np.ndarray, window: int, hop_length: int) -> np.ndarray:
    """dsp.py:11-25"""
    idx = np.arange(window)[:, None] + np.arange((len(a) - window) // hop_length + 1)[None, :] * hop_length
    return a[idx]


def mel_filter(y: np.ndarray, n_fft=1024, sr=16000, n_mels=80, fmin=0.0, fmax=8000.0, dtype=np.float32) -> np.ndarray:
    """MelFilter.__call__ (dsp.py:115-128).  y [B,S] -> log-mel [B,F,80].
    dtype float32 mirrors the reference's precision (complex64 FFT); float64 is
    the arbiter."""
    assert y.ndim == 2
    cdtype = np.complex64 if dtype == np.float32 else np.complex128
    melfb = librosa_mel_filterbank(sr, n_fft, n_mels, fmin, fmax).astype(dtype)
    hop = n_fft // 4
    y = np.asarray(y, dtype).T  # n s -> s n
    p = (n_fft - hop) // 2
    y = np.pad(y, ((p, p), (0, 0)), mode="reflect")
    window = np.hanning(n_fft + 1)[:-1].astype(dtype)
    frames = rolling_window(y, n_fft, hop) * window[:, None, None]  # [1024, F, B]
    spec = np.fft.fft(frames.astype(cdtype), axis=0)[: 1 + n_fft // 2].astype(cdtype)
    mag = np.sqrt(np.square(spec.real) + np.square(spec.imag) + dtype(1e-9)).astype(dtype)
    mel = np.einsum("ms,sfn->nfm", melfb, mag).astype(dtype)
    return np.log(np.clip(mel, 1e-5, None)).astype(dtype)
