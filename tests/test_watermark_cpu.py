"""CPU: the watermark's definition (oracle/watermark_oracle.py), the tolerances the GPU tests hold it to, its null
bound and its robustness on real speech.

TOL_EMBED bounds |y - y64| per output in units of denoise_oracle.error_scale (the denoiser's fp32 error scale of the
same STFT), TOL_Z bounds |z - z64|.  Each is a few times the worst fp32 emulation of the kernels (the kernels' order of
operations, fp32 torch FFTs), and each wrong variant of the definition exceeds it by orders of magnitude."""
from pathlib import Path

import numpy as np
import pytest
import scipy.signal as ss
import torch

from oracle import denoise_oracle as dn
from oracle import watermark_oracle as wo
from viettts_b200 import jaxrng

SR = 16000
TOL_EMBED = 2e-7     # per output, relative to error_scale (see test_tolerances_have_headroom_over_the_emulation)
TOL_Z = 2e-3         # absolute, on z
KEY = 7
WRONG_KEYS = list(range(1000, 1064))
CLIP = Path(__file__).resolve().parent / "golden" / "watermark_speech_clip.npz"


def speech(seconds=20.0, start=0.0):
    """float64 excerpt of the fixture: 20 s of real speech as int16 at 16 kHz"""
    pcm = np.load(CLIP)["pcm"]
    return pcm[int(start * SR): int((start + seconds) * SR)].astype(np.float64) / 32768.0


def embed_scale(x, eps):
    return dn.error_scale(x, 0.0, np.zeros(dn.N_BINS)) * (1.0 + eps)


# ---- fp32 emulation of the kernels ----
def _spectra(x, hop):
    x = np.asarray(x, np.float32)
    w = dn.window().astype(np.float32)
    xp = np.pad(x, dn.PAD, mode="reflect")
    T = x.size // hop + 1
    idx = hop * np.arange(T)[:, None] + np.arange(dn.N_FFT)[None, :]
    return torch.fft.fft(torch.from_numpy(xp[idx] * w).to(torch.complex64), dim=1)[:, : dn.N_BINS]


def emulate_embed(x, key, eps, group_shift=0, k0=wo.K0, sign=1.0):
    """the embed kernels in fp32; variants: chips of group j + group_shift, the band starting at k0, gain 1 - eps c"""
    x = np.asarray(x, np.float32)
    n = x.size
    if n <= dn.PAD or eps == 0:
        return x.copy()
    X = _spectra(x, dn.HOP)
    F = X.shape[0]
    c = wo.chips(key)
    j = ((np.arange(F) + wo.G * group_shift) // wo.G) % wo.P
    gain = np.ones((F, dn.N_BINS), np.float32)
    up, down = np.float32(1) + np.float32(eps), np.float32(1) - np.float32(eps)
    cc = c[j][:, : wo.K1 - k0] * sign
    gain[:, k0: wo.K1] = np.where(cc < 0, down, up)
    Y = X * torch.from_numpy(gain)
    full = torch.cat([Y, torch.conj(Y[:, 1: dn.N_BINS - 1]).flip(1)], dim=1)
    w = dn.window().astype(np.float32)
    yf = (torch.fft.fft(torch.conj(full), dim=1).real.numpy() * np.float32(1.0 / dn.N_FFT)) * w
    acc = np.zeros(dn.N_FFT + dn.HOP * (F - 1), np.float32)
    env = np.zeros_like(acc)
    w2 = w.astype(np.float64) ** 2
    for f in range(F):
        sl = slice(dn.HOP * f, dn.HOP * f + dn.N_FFT)
        acc[sl] = acc[sl] + yf[f]
        env[sl] = (w2 + env[sl].astype(np.float64)).astype(np.float32)
    return acc[dn.PAD: dn.PAD + n] / env[dn.PAD: dn.PAD + n]


def emulate_z(x, keys, neighbours=True):
    """z [K, 64, 16] of the detect kernels in fp32; variant: no neighbour-group subtraction"""
    X = _spectra(x, wo.DET_HOP)
    re, im = X.real.numpy(), X.imag.numpy()
    M = np.log(re * re + im * im + np.float32(1e-12)).astype(np.float32)[:, wo.K0 - 4: wo.K1 + 4]
    s = np.zeros((M.shape[0], wo.NK), np.float32)
    for d in range(9):
        s = s + M[:, d: d + wo.NK]
    D = M[:, 4: 4 + wo.NK] - s * np.float32(1.0 / 9.0)
    C = np.stack([wo.chips(k) for k in keys]).astype(np.float32)
    z = np.zeros((len(keys), wo.P, wo.NQ))
    for q in range(wo.NQ):
        Dq = D[q::4]
        ng = Dq.shape[0] // wo.G
        Gs = ((Dq[0: 4 * ng: 4] + Dq[1: 4 * ng: 4]) + Dq[2: 4 * ng: 4]) + Dq[3: 4 * ng: 4]
        H = np.zeros_like(Gs)
        if ng > 2:
            H[1:-1] = Gs[1:-1] - np.float32(0.5) * (Gs[:-2] + Gs[2:]) if neighbours else Gs[1:-1]
        S = np.zeros((wo.P, wo.NK), np.float32)
        for g in range(ng):
            S[g % wo.P] += H[g]
        den = np.sqrt(np.sum(S.astype(np.float32) ** 2, dtype=np.float32))
        A = np.einsum("jk,cmk->cjm", S, C)
        for p in range(wo.P):
            z[:, p, q] = A[:, np.arange(wo.P), (np.arange(wo.P) + p) % wo.P].sum(axis=1) / den
    return z


# ---- definition ----
def test_chips_equal_jaxrng_threefry():
    for key in (0, 7, 2 ** 32 + 5, 2 ** 64 - 1):
        j, k = np.meshgrid(np.arange(wo.P), np.arange(wo.K0, wo.K1), indexing="ij")
        o0, _ = jaxrng.threefry2x32(key & 0xFFFFFFFF, key >> 32, j.ravel().astype(np.uint32), k.ravel().astype(np.uint32))
        assert np.array_equal(np.where(o0 >> 31, -1.0, 1.0).reshape(wo.P, wo.NK), wo.chips(key)), key


def test_band_period_and_edge_cases():
    assert wo.K0 * SR / dn.N_FFT == 312.5 and (wo.K1 - 1) * SR / dn.N_FFT < 3422
    assert wo.PERIOD == 65536
    x = speech(2.0)
    assert np.array_equal(wo.embed(x, KEY, 0.0), x)
    assert np.array_equal(wo.embed(x[:512], KEY, 0.2), x[:512])
    assert np.array_equal(wo.embed(np.zeros(5000), KEY, 0.2), np.zeros(5000))
    z, off = wo.detect(np.zeros(20000), [KEY])
    assert z[0] == 0 and off[0] == 0
    assert wo.detect(x[:512], [KEY])[0][0] == 0


def test_tolerances_have_headroom_over_the_emulation():
    x = speech(6.0, 3.0)
    worst = 0.0
    for n, eps in ((513, 0.1), (1024, 0.3), (40000, 0.1), (x.size, 0.05)):
        n = int(n)
        ref = wo.embed(x[:n], KEY, eps)
        e = np.max(np.abs(emulate_embed(x[:n], KEY, eps) - ref) / embed_scale(x[:n], eps))
        worst = max(worst, e)
    variants = [emulate_embed(x, KEY, 0.1, group_shift=1), emulate_embed(x, KEY, 0.1, k0=wo.K0 + 1),
                emulate_embed(x, KEY, 0.1, sign=-1.0)]
    ref = wo.embed(x, KEY, 0.1)
    wrong = [np.max(np.abs(v - ref) / embed_scale(x, 0.1)) for v in variants]
    print(f"embed: fp32 emulation {worst:.2e}, variants {', '.join(f'{w:.1e}' for w in wrong)} (TOL {TOL_EMBED:.0e})")
    assert 4 * worst <= TOL_EMBED and min(wrong) >= 100 * TOL_EMBED

    y = wo.embed(x, KEY, 0.1).astype(np.float32)
    keys = [KEY, 8]
    zref = wo.scores(y, keys)
    zem = emulate_z(y, keys)
    worst_z = np.max(np.abs(zem - zref))
    wrong_z = np.max(np.abs(emulate_z(y, keys, neighbours=False) - zref))
    # a mark on the wrong group or band scores near zero against the right one
    shifted = wo.scores(emulate_embed(x, KEY, 0.1, group_shift=1), keys, search=False)[0, 0, 0]
    flipped = wo.scores(emulate_embed(x, KEY, 0.1, sign=-1.0), keys, search=False)[0, 0, 0]
    print(f"z: fp32 emulation {worst_z:.2e}, no neighbour subtraction {wrong_z:.2e}, aligned z {zref[0, 0, 0]:.2f}, "
          f"group shifted {shifted:.2f}, sign flipped {flipped:.2f} (TOL {TOL_Z:.0e})")
    assert 4 * worst_z <= TOL_Z and wrong_z >= 100 * TOL_Z
    assert zref[0, 0, 0] - shifted >= 100 * TOL_Z and zref[0, 0, 0] - flipped >= 100 * TOL_Z


def test_search_finds_a_crop_and_its_offset():
    """the offset comes back to within one search step (64 samples): frames 64 samples off the embedder's still carry
    most of the mark"""
    y = wo.embed(speech(), KEY, 0.1)
    for c in (0, 64 * 193, 64 * 1000 + 3 * 1024, 65536 + 640):
        z, off = wo.detect(y[c: c + 5 * SR], [KEY])
        d = (int(off[0]) - c) % 65536
        assert z[0] >= wo.SEARCH_THRESHOLD and min(d, 65536 - d) <= wo.DET_HOP, (c, z, off)


# ---- null bound ----
def null_signals():
    rng = np.random.default_rng(5)
    n = 6 * SR
    t = np.arange(n) / SR
    white = 0.1 * rng.standard_normal(n)
    b, a = [0.049922, -0.095993, 0.050612, -0.004408], [1, -2.494956, 2.017265, -0.522190]
    pink = ss.lfilter(b, a, rng.standard_normal(n))
    tones = 0.3 * np.sin(2 * np.pi * 440 * t) + 0.2 * np.sin(2 * np.pi * 1234.5 * t)
    clicks = np.zeros(n)
    clicks[::4000] = 0.9
    out = {"white": white, "pink": pink, "tones": tones, "clicks": clicks, "silence": np.zeros(n)}
    for s in (0.0, 7.3, 13.0):
        out[f"speech@{s}"] = speech(6.0, s)
    out["marked speech, other keys"] = wo.embed(speech(6.0, 2.0), KEY, 0.3)
    return out


def test_null_bound_with_64_wrong_keys():
    """For audio without the key, z at one offset is a Rademacher sum: P(z >= tau) <= exp(-tau^2 / 2).  Over every
    signal, 64 wrong keys and all 1024 offsets (about 6e5 scores) the tail stays under that bound, no aligned score
    reaches 5 and no search maximum reaches 6.5.  (The largest of 6e5 such scores is expected near
    sqrt(2 ln 6e5) = 5.2, so search maxima over many keys do come close to 5.)"""
    worst = worst_aligned = 0.0
    allz = []
    for name, x in null_signals().items():
        z = wo.scores(x, WRONG_KEYS)
        allz.append(z.ravel())
        worst, worst_aligned = max(worst, float(z.max())), max(worst_aligned, float(np.abs(z[:, 0, 0]).max()))
        assert z.max() < wo.SEARCH_THRESHOLD and np.abs(z[:, 0, 0]).max() < wo.ALIGNED_THRESHOLD, (name, z.max())
    allz = np.concatenate(allz)
    for tau in (2.0, 3.0, 4.0):
        assert np.mean(allz >= tau) <= np.exp(-tau * tau / 2), tau
    print(f"{allz.size} wrong-key scores: largest {worst:.2f}, largest aligned |z| {worst_aligned:.2f}")


# ---- robustness on real speech (float64, the issue's feasibility numbers within 30 %) ----
def butter_sos(order, f, kind):
    return ss.butter(order, f, kind, fs=SR, output="sos")


def test_robustness_on_the_fixture():
    from viettts_b200.engine import reverb_params
    x = speech()
    y = wo.embed(x, KEY, 0.1)
    hp, lp = butter_sos(4, 300, "highpass"), butter_sos(4, 3400, "lowpass")

    def rev(v, spec):
        p = reverb_params(spec, SR)
        return (1 - p["mix"]) * v + p["mix"] * ss.fftconvolve(v, p["ir"].astype(np.float64))[: v.size]

    stages = {
        "nothing": (lambda v: v, 15.7),
        "pcm16": (lambda v: np.round(v * 32767) / 32767, 13.6),
        "48k": (lambda v: ss.resample_poly(ss.resample_poly(v, 3, 1), 1, 3), 15.7),
        "8k": (lambda v: ss.resample_poly(ss.resample_poly(v, 1, 2), 2, 1), 15.7),
        "telephone": (lambda v: ss.sosfilt(lp, ss.sosfilt(hp, v)), 15.8),
        "room": (lambda v: rev(v, "room"), 11.5),
    }
    for name, (f, expect) in stages.items():
        z = wo.detect(f(y), [KEY], search=False)[0][0]
        print(f"{name}: z {z:.1f} (feasibility {expect})")
        assert 0.7 * expect <= z <= 1.3 * expect, (name, z)
    assert abs(wo.detect(y, [8], search=False)[0][0]) <= 1.0
    snr = 10 * np.log10(np.sum(x * x) / np.sum((y - x) ** 2))
    assert 24.8 - 3 <= snr <= 24.8 + 3, snr
