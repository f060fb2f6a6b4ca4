"""Float64 statement of the watermark (vtts_watermark*, vtts_watermark_detect*): a keyed spread-spectrum mark on the
denoiser's STFT and its detector.

Embed, one 16 kHz row x of n samples, key kappa (uint64), strength eps in [0, 0.3]:
    STFT   the denoiser's (denoise_oracle: n_fft 1024, hop 256, periodic Hann, centered frames, reflect padding 512)
    chips  c(kappa, j, k) = -1 where the top bit of word 0 of threefry2x32(kappa_lo, kappa_hi, j, k) is set, else +1
    gain   Y_f[k] = X_f[k] (1 + eps c(kappa, j, k)) for k in [20, 219), j = floor(f / 4) mod 64; other bins unchanged
    ISTFT  the denoiser's overlap-add; n <= 512 and eps = 0 return x unchanged
Detect, one 16 kHz row, keys kappa_1..K:
    D      log(|X_t|^2 + 1e-12) of the hop-64 frames (same centered framing), less its 9-bin moving mean across
           frequency, on the band
    fold   per frame phase q in [0, 16): hop-256 frames f at t = q + 4 f; group sums G_g of 4 of them;
           H_g = G_g - (G_{g-1} + G_{g+1}) / 2, 0 for the first and last group; S_j = sum over g = j mod 64 of H_g
    z      z(p, q) = sum_{j,k} S_j[k] c(kappa, (j + p) mod 64, k) / sqrt(sum S^2), 0 when the denominator is 0
    Aligned mode reads z(0, 0), offset 0.  Search mode: the largest z over the 1024 (p, q), the first in ascending
    offset (1024 p - 64 q) mod 65536 among equal ones; the offset is where the row's sample 0 sits in the mark's period.
    Rows of n <= 512 give z = 0.
"""
from __future__ import annotations

import numpy as np

from oracle import denoise_oracle as dn

K0, K1 = 20, 219              # band bins [K0, K1): 312.5 .. 3421.9 Hz
NK = K1 - K0
G, P = 4, 64                  # hop-256 frames per chip group, groups per period
NQ = 16                       # frame phases of the search
DET_HOP = 64
FLOOR = 1e-12
PERIOD = P * G * dn.HOP       # 65536 samples
MAX_STRENGTH = 0.3
ALIGNED_THRESHOLD, SEARCH_THRESHOLD = 5.0, 6.5

_ROT = ((13, 15, 26, 6), (17, 29, 16, 24))
_M32 = 0xFFFFFFFF


def threefry2x32(k0: int, k1: int, c0: int, c1: int):
    """Threefry-2x32, 20 rounds, on Python integers (one counter pair)."""
    ks = (k0, k1, 0x1BD11BDA ^ k0 ^ k1)
    x0, x1 = (c0 + k0) & _M32, (c1 + k1) & _M32
    for blk in range(5):
        for r in _ROT[blk & 1]:
            x0 = (x0 + x1) & _M32
            x1 = (((x1 << r) | (x1 >> (32 - r))) & _M32) ^ x0
        x0 = (x0 + ks[(blk + 1) % 3]) & _M32
        x1 = (x1 + ks[(blk + 2) % 3] + blk + 1) & _M32
    return x0, x1


_chip_cache: dict = {}


def chips(key: int) -> np.ndarray:
    """c(key, j, k) as float64 [64, 199] (j, k - 20)"""
    key = int(key)
    if key not in _chip_cache:
        lo, hi = key & _M32, key >> 32
        c = np.empty((P, NK))
        for j in range(P):
            for k in range(K0, K1):
                c[j, k - K0] = -1.0 if threefry2x32(lo, hi, j, k)[0] >> 31 else 1.0
        _chip_cache[key] = c
    return _chip_cache[key]


def embed(x, key: int, eps: float, frame0: int = 0) -> np.ndarray:
    """y of one row in float64 (x taken as float64).  `frame0` is the absolute index of the row's frame 0: a row that
    starts at sample 256 frame0 of a stream slot, so chip group j = floor((frame0 + f) / 4) mod 64 keys its frame f"""
    x = np.asarray(x, np.float64)
    n = x.size
    if n <= dn.PAD or eps == 0:
        return x.copy()
    X = dn.stft(x)
    f = int(frame0) + np.arange(X.shape[0], dtype=np.int64)
    X[:, K0:K1] *= 1.0 + float(eps) * chips(key)[(f // G) % P]
    y = np.fft.irfft(X, dn.N_FFT, axis=1) * dn.window()[None, :]
    return dn.overlap_add(y, n) / dn.envelope(n)


def whitened(x) -> np.ndarray:
    """D [T, 199] of one row (n > 512): the whitened band of its hop-64 frames"""
    x = np.asarray(x, np.float64)
    xp = np.pad(x, dn.PAD, mode="reflect")
    T = x.size // DET_HOP + 1
    idx = DET_HOP * np.arange(T)[:, None] + np.arange(dn.N_FFT)[None, :]
    X = np.fft.rfft(xp[idx] * dn.window(), axis=1)
    M = np.log(np.abs(X[:, K0 - 4: K1 + 4]) ** 2 + FLOOR)
    mean = sum(M[:, d: d + NK] for d in range(9)) / 9.0
    return M[:, 4: 4 + NK] - mean


def fold(D, q: int) -> np.ndarray:
    """S [64, 199] of frame phase q"""
    Dq = D[q::4]
    ng = Dq.shape[0] // G
    Gs = Dq[: ng * G].reshape(ng, G, NK).sum(axis=1)
    H = np.zeros_like(Gs)
    if ng > 2:
        H[1:-1] = Gs[1:-1] - 0.5 * (Gs[:-2] + Gs[2:])
    S = np.zeros((P, NK))
    np.add.at(S, np.arange(ng) % P, H)
    return S


def offset_of(p: int, q: int) -> int:
    return (1024 * p - DET_HOP * q) % PERIOD


def scores(x, keys, search: bool = True) -> np.ndarray:
    """z [K, 64, 16] (search) or [K, 1, 1] over (p, q) of one 16 kHz row"""
    x = np.asarray(x, np.float64)
    nq, npp = (NQ, P) if search else (1, 1)
    z = np.zeros((len(keys), npp, nq))
    if x.size <= dn.PAD:
        return z
    D = whitened(x)
    C = np.stack([chips(k) for k in keys])                # [K, 64, 199]
    for q in range(nq):
        S = fold(D, q)
        den = np.sqrt(np.sum(S * S))
        if den == 0:
            continue
        A = np.einsum("jk,cmk->cjm", S, C)               # [K, j, m]
        for p in range(npp):
            z[:, p, q] = A[:, np.arange(P), (np.arange(P) + p) % P].sum(axis=1) / den
    return z


def detect(x, keys, search: bool = True):
    """(z [K], offset [K]) of one 16 kHz row: z(0, 0) aligned, else the maximum over the 1024 offsets and its offset"""
    z = scores(x, keys, search)
    best = np.zeros(len(keys))
    off = np.zeros(len(keys), np.int64)
    for c in range(len(keys)):
        cand = sorted(((-z[c, p, q], offset_of(p, q)) for p in range(z.shape[1]) for q in range(z.shape[2])))
        best[c], off[c] = -cand[0][0], cand[0][1]
    return best, off
