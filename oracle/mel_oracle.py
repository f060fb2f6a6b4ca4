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


def mel_linear(y: np.ndarray, n_fft=1024, sr=16000, n_mels=80, fmin=0.0, fmax=8000.0, dtype=np.float32, fb=None) -> np.ndarray:
    """MelFilter.__call__ (dsp.py:115-126) before the clip and the log: y [B,S] -> mel [B,F,80].  fb
    [n_mels, 1+n_fft//2] replaces the Slaney bank of (sr, fmin, fmax)."""
    assert y.ndim == 2
    cdtype = np.complex64 if dtype == np.float32 else np.complex128
    melfb = (librosa_mel_filterbank(sr, n_fft, n_mels, fmin, fmax) if fb is None else np.asarray(fb, np.float32)).astype(dtype)
    hop = n_fft // 4
    y = np.asarray(y, dtype).T  # n s -> s n
    p = (n_fft - hop) // 2
    y = np.pad(y, ((p, p), (0, 0)), mode="reflect")
    window = np.hanning(n_fft + 1)[:-1].astype(dtype)
    frames = rolling_window(y, n_fft, hop) * window[:, None, None]  # [1024, F, B]
    spec = np.fft.fft(frames.astype(cdtype), axis=0)[: 1 + n_fft // 2].astype(cdtype)
    mag = np.sqrt(np.square(spec.real) + np.square(spec.imag) + dtype(1e-9)).astype(dtype)
    return np.einsum("ms,sfn->nfm", melfb, mag).astype(dtype)


def mel_filter(y: np.ndarray, n_fft=1024, sr=16000, n_mels=80, fmin=0.0, fmax=8000.0, dtype=np.float32, fb=None) -> np.ndarray:
    """MelFilter.__call__ (dsp.py:115-128).  y [B,S] -> log-mel [B,F,80].
    dtype float32 mirrors the reference's precision (complex64 FFT); float64 is
    the arbiter.  fb [n_mels, 1+n_fft//2] replaces the Slaney bank of (sr, fmin, fmax)."""
    mel = mel_linear(y, n_fft, sr, n_mels, fmin, fmax, dtype, fb)
    return np.log(np.clip(mel, 1e-5, None)).astype(dtype)


# ---- fp32 emulation of csrc/melspec.cu, and the error scale the kernel is held to ----------------------------------
#
# melspec_kernel runs one warp per frame pair (2j, 2j+1): frame A is the real part and frame B the imaginary part of
# one complex FFT-1024, factored 32 x 32 (pass 1 over m of the samples n = l + 32 m, the inter-pass twiddles, pass 2
# over l), then separated into the two real spectra.  `emulate` repeats that arithmetic in float32 numpy, operation for
# operation; it differs from the device only where nvcc contracts a product and a sum into one fma and where
# sqrt.approx.f32 and logf round differently from numpy (each well under one unit of the error scale below).

NFFT, HOP, PAD, NB = 1024, 256, 384, 513
LOG_CLIP = np.log(np.float32(1e-5))      # log(max(mel, 1e-5)) of every bin whose filterbank sum is below the clip


def _bitrev5(x):
    return ((x & 1) << 4) | ((x & 2) << 2) | (x & 4) | ((x & 8) >> 2) | ((x & 16) >> 4)


_BR = _bitrev5(np.arange(32))
_W32 = np.exp(-2j * np.pi * np.arange(16) / 32)
_W32R, _W32I = _W32.real.astype(np.float32), _W32.imag.astype(np.float32)


def _cmul(ar, ai, br, bi):
    """fftc::cmul: each product and sum rounded to float32"""
    return ar * br - ai * bi, ar * bi + ai * br


def _fft32(re, im):
    """fftc::fft32 along the last axis: radix-2 decimation in frequency; on return [..., p] holds X[bitrev5(p)]"""
    lead = re.shape[:-1]
    for half in (16, 8, 4, 2, 1):
        re = re.reshape(*lead, 32 // (2 * half), 2, half)
        im = im.reshape(*lead, 32 // (2 * half), 2, half)
        ar, br, ai, bi = re[..., 0, :], re[..., 1, :], im[..., 0, :], im[..., 1, :]
        dr, di = ar - br, ai - bi
        tk = np.arange(half) * (16 // half)             # W_{2 half}^j = W_32^tk
        mr, mi = _cmul(dr, di, _W32R[tk], _W32I[tk])
        mr = np.where(tk == 0, dr, np.where(tk == 8, di, mr))     # W^0 = 1 and W^8 = -i are not multiplied
        mi = np.where(tk == 0, di, np.where(tk == 8, -dr, mi))
        re = np.stack([ar + br, mr], axis=-2).reshape(*lead, 32)
        im = np.stack([ai + bi, mi], axis=-2).reshape(*lead, 32)
    return re, im


def _twiddles(extra_step=False):
    """[l, k1] = w1^k1 with w1 = exp(-2 pi i l / 1024) in float32, as four interleaved power chains of w4 = w1^4
    (r[c] = w1^(4 q + c)).  extra_step: chain 3 steps once more than it should (a mutation for the tests)."""
    a = -2.0 * np.pi * np.arange(32) / NFFT
    w1 = (np.cos(a).astype(np.float32), np.sin(a).astype(np.float32))
    w2 = _cmul(*w1, *w1)
    w3 = _cmul(*w2, *w1)
    w4 = _cmul(*w2, *w2)
    r = [(np.ones(32, np.float32), np.zeros(32, np.float32)), w1, w2, w3]
    tr, ti = np.zeros((32, 32), np.float32), np.zeros((32, 32), np.float32)
    for q in range(8):
        for c in range(4):
            tr[:, 4 * q + c], ti[:, 4 * q + c] = r[c]
            if q < 7:
                r[c] = _cmul(*r[c], *w4)
                if extra_step and c == 3 and q == 6:
                    r[c] = _cmul(*r[c], *w4)
    return tr, ti


def _pair_rows(y, pad="reflect"):
    """The 1280 samples the warp of each frame pair reads: [B, P, 1280], sample t of pair j at input index
    512 j - 384 + t, reflected about the first and last sample (dsp.py:119-121); frame A is t < 1024, frame B is
    t >= 256.  A lone last frame (odd F) pairs with zeros past t = 1024.  pad="symmetric" repeats the edge sample
    instead (a mutation for the tests)."""
    B, S = y.shape
    F = S // HOP
    i = 2 * HOP * np.arange((F + 1) // 2)[:, None] - PAD + np.arange(NFFT + HOP)[None, :]
    if pad == "reflect":
        i = np.where(i < 0, -i, np.where(i >= S, 2 * (S - 1) - i, i))
    else:
        i = np.where(i < 0, -1 - i, np.where(i >= S, 2 * S - 1 - i, i))
    raw = y[:, np.clip(i, 0, S - 1)]
    if F % 2:
        raw[:, -1, NFFT:] = 0
    return raw


def _hann(dtype):
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(NFFT) / NFFT)).astype(dtype)   # np.hanning(1025)[:-1], dsp.py:81


def mel_spans(fb):
    """mel_span_kernel's rule: row m of the bank is summed over [lo[m], hi[m]), from its first to one past its last
    non-zero entry; lo = hi = 0 for an all-zero row"""
    fb = np.asarray(fb, np.float32)
    lo, hi = np.zeros(len(fb), np.int64), np.zeros(len(fb), np.int64)
    for m, row in enumerate(fb):
        nz = np.flatnonzero(row != 0)
        if nz.size:
            lo[m], hi[m] = nz[0], nz[-1] + 1
    return lo, hi


def emulate(y, fb, pad="reflect", drop_last_bin=False, b_mirror_sign=False, chain_extra_step=False) -> np.ndarray:
    """melspec_kernel in float32: y [B,S] (S a multiple of 256, >= 512) and the bank fb [80,513] -> log-mel [B,F,80].
    The keyword arguments are mutations the tests must be able to see: symmetric padding, a span one bin short, frame
    B's real part taking the mirrored bin's imaginary part with the wrong sign, a power chain one step long."""
    y = np.asarray(y, np.float32)
    B, S = y.shape
    F = S // HOP
    raw = _pair_rows(y, pad)
    P = raw.shape[1]
    h = _hann(np.float32)
    a, b = raw[..., :NFFT] * h, raw[..., HOP:] * h
    # pass 1: lane l holds n = l + 32 m; DFT over m, then the twiddle w1^k1 (k1 = 0 stored as is)
    re, im = _fft32(a.reshape(B, P, 32, 32).swapaxes(-1, -2), b.reshape(B, P, 32, 32).swapaxes(-1, -2))
    re, im = re[..., _BR], im[..., _BR]
    tr, ti = _twiddles(chain_extra_step)
    yr, yi = _cmul(re, im, tr, ti)
    yr[..., 0], yi[..., 0] = re[..., 0], im[..., 0]
    # pass 2: lane k1, DFT over l: Z[k1 + 32 k2]
    re, im = _fft32(yr.swapaxes(-1, -2), yi.swapaxes(-1, -2))
    zr = re[..., _BR].swapaxes(-1, -2).reshape(B, P, NFFT)
    zi = im[..., _BR].swapaxes(-1, -2).reshape(B, P, NFFT)
    # separation A = (Z[k] + conj Z[N-k]) / 2, B = (Z[k] - conj Z[N-k]) / 2i, and the magnitudes
    k = np.arange(NB)
    kc = (NFFT - k) & (NFFT - 1)
    z_r, z_i, c_r, c_i = zr[..., k], zi[..., k], zr[..., kc], zi[..., kc]
    half, eps = np.float32(0.5), np.float32(1e-9)
    ar, ai = half * (z_r + c_r), half * (z_i - c_i)
    br, bi = half * ((z_i - c_i) if b_mirror_sign else (z_i + c_i)), -half * (z_r - c_r)
    mags = (np.sqrt(ar * ar + ai * ai + eps), np.sqrt(br * br + bi * bi + eps))
    # the filterbank over each row's span, one fmaf per bin in increasing k, then log(max(., 1e-5))
    fb = np.asarray(fb, np.float32)
    M = fb.shape[0]
    lo, hi = mel_spans(fb)
    if drop_last_bin:
        hi = np.maximum(hi - 1, lo)
    out = np.empty((B, F, M), np.float32)
    for ch, mag in enumerate(mags):
        s = np.zeros((B, P, M), np.float32)
        for j in range(int((hi - lo).max())):
            kk = np.minimum(lo + j, NB - 1)
            t = (fb[np.arange(M), kk].astype(np.float64) * mag[..., kk] + s).astype(np.float32)   # fmaf: one rounding
            s = np.where(lo + j < hi, t, s)
        out[:, ch::2] = np.log(np.maximum(s, np.float32(1e-5)))[:, : (F + 1 - ch) // 2]
    return out


def mel_error_scale(y, fb):
    """(scale, m64): the float64 mel m64 [B,F,80] (before the clip) and the error scale [B,F,80] of an fp32 log-mel,

        2^-24 (log2(1024) ||w x_pair||_2 sum_k fb[m,k] + (1 + |log m_ref|) m_ref),   m_ref = max(m64, 1e-5)

    FFT round-off spreads over every bin in proportion to the norm of the transformed sequence, so a bin's error does
    not shrink with its own energy; the sequence is the packed pair a + i b, so ||w x_pair||^2 = ||w a||^2 + ||w b||^2
    over the two frames of the warp (a quiet frame next to a loud one carries the loud one's round-off).  Each
    filterbank weight takes that error once.  The second term is the sum's relative rounding and the log's: a float32
    log rounds to half an ulp of |log m|, which is |log m| 2^-24 relative once exponentiated."""
    y = np.asarray(y, np.float64)
    F = y.shape[1] // HOP
    raw = _pair_rows(y)
    h = _hann(np.float64)
    n2 = ((raw[..., :NFFT] * h) ** 2).sum(-1) + ((raw[..., HOP:] * h) ** 2).sum(-1)
    norm = np.repeat(np.sqrt(n2), 2, axis=1)[:, :F]
    fb = np.asarray(fb, np.float32)
    m64 = mel_linear(y, dtype=np.float64, fb=fb)
    m_ref = np.maximum(m64, 1e-5)
    scale = 2.0 ** -24 * (np.log2(NFFT) * norm[..., None] * fb.astype(np.float64).sum(1) + (1 + np.abs(np.log(m_ref))) * m_ref)
    return scale, m64


def mel_error(got, y, fb, tol):
    """(units, bad_clip): |exp(got) - max(m64, 1e-5)| / scale per bin [B,F,80] (inf where got is not finite), and the
    number of bins that are below log(1e-5), or that float64 puts below the clip by more than tol units and that are
    not log(1e-5) bit for bit"""
    got = np.asarray(got, np.float32)
    scale, m64 = mel_error_scale(y, fb)
    units = np.abs(np.exp(got.astype(np.float64)) - np.maximum(m64, 1e-5)) / scale
    units = np.where(np.isfinite(got), units, np.inf)
    must_clip = m64 + tol * scale <= 1e-5
    bad_clip = int(np.count_nonzero((got < LOG_CLIP) | (must_clip & (got != LOG_CLIP))))
    return units, bad_clip
