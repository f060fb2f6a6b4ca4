"""CPU: the voice shifter's definition (oracle/voice_shift_oracle.py), the tolerance the GPU tests hold it to, and what
the Python layer hands to the library.

The oracle is checked on what a formant control must do: the envelope warp an LPC estimator sees in the output is f
(the formant ratio) in every case with a formant shift, and r (the pitch ratio) without one, while the output's F0 stays
r F0.  TOL_F -- the bound |y - y64| <= TOL_F * voice_shift_oracle.error_scale per output -- comes from an fp32
emulation of the kernels in their reduction order, run under float64's decisions, as test_pitch_cpu.py derives TOL."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from oracle import denoise_oracle as do
from oracle import pitch_oracle as po
from oracle import voice_shift_oracle as vo
from test_denoise_cpu import signal_of, to_bf16
from test_pitch_cpu import voiced_of

SR = 16000
TOL_F = 9e-6    # per output, relative to vo.error_scale (see test_bound_has_headroom_over_the_emulation)
CLIP = Path(__file__).resolve().parent / "golden" / "watermark_speech_clip.npz"


# ---- signals and the envelope-warp estimator -------------------------------------------------------------------

def vowel(f0, seconds=1.0, seed=0):
    """a pulse train at f0 with 0.3 % period jitter through resonators at 700 / 1220 / 2600 Hz (bandwidths 80 / 90 /
    120 Hz), peak 0.5"""
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    x = np.zeros(n)
    t = 0.0
    while t < n:
        x[int(t)] = 1.0
        t += SR / f0 * (1 + 0.003 * rng.standard_normal())
    for F, bw in ((700, 80), (1220, 90), (2600, 120)):
        rr = np.exp(-np.pi * bw / SR)
        x = lfilter([1.0], [1.0, -2 * rr * np.cos(2 * np.pi * F / SR), rr * rr], x)
    return (0.5 * x / np.abs(x).max()).astype(np.float32)


def speech(seconds=6.0):
    d = np.load(CLIP)
    assert int(d["rate"]) == SR
    return (d["pcm"][: int(seconds * SR)].astype(np.float64) / 32768.0).astype(np.float32)


GRID = np.arange(50.0, 7900.0 + 1e-9, 5.0)     # Hz


def lpc_envelope(x, order=18):
    """the mean LPC log-envelope (dB on GRID) of the Hann frames of 512 at hop 256 whose RMS is >= 0.3 of the largest"""
    x = np.asarray(x, np.float64)
    w = np.hanning(512)
    starts = range(0, x.size - 512 + 1, 256)
    fr = np.stack([x[s: s + 512] * w for s in starts])
    rms = np.sqrt((fr ** 2).mean(axis=1))
    fr = fr[rms >= 0.3 * rms.max()]
    env = []
    z = np.exp(-2j * np.pi * np.outer(GRID / SR, np.arange(order + 1)))
    for f in fr:
        r = np.correlate(f, f, "full")[f.size - 1: f.size + order]
        a, err = np.array([1.0]), r[0]
        for i in range(1, order + 1):                       # Levinson-Durbin
            k = -(r[i] + a[1:] @ r[i - 1: 0: -1]) / err
            a = np.concatenate([a, [0.0]]) + k * np.concatenate([a, [0.0]])[::-1]
            err *= 1 - k * k
        env.append(10 * np.log10(max(err, 1e-30)) - 20 * np.log10(np.abs(z @ a)))
    return np.mean(env, axis=0)


def warp_steps(x, y):
    """j of the warp w = 2^(j / 48), j in [-48, 48], that best maps the input's envelope onto the output's: the largest
    correlation of E_y(nu) with E_x(nu / w) over 200..4000 Hz"""
    ex, ey = lpc_envelope(x), lpc_envelope(y)
    band = (GRID >= 200) & (GRID <= 4000)
    nu = GRID[band]
    best = max(range(-48, 49), key=lambda j: np.corrcoef(ey[band], np.interp(nu / 2 ** (j / 48), GRID, ex))[0, 1])
    return best


def f0_of(y, lo=60.0, hi=500.0):
    """F0 of a steady stretch by autocorrelation with a parabolic peak"""
    y = np.asarray(y, np.float64)
    y = y - y.mean()
    ac = np.correlate(y, y, "full")[y.size - 1:]
    a, b = int(SR / hi), int(SR / lo)
    i = a + int(np.argmax(ac[a:b]))
    p, q, r = ac[i - 1: i + 2]
    return SR / (i + 0.5 * (p - r) / (p - 2 * q + r))


# cases: (s, phi) -> the warp the output must show (in steps of 1/48 octave) and how far off it may be
KEEP_MOVE = [(3, 0), (-3, 0), (7, 0), (-7, 0), (0, 3), (0, -3), (5, -2)]
LEGACY = [(3, None), (-7, None)]


def expected_steps(s, phi):
    return 48 * np.log2(float(po.ratio(s))) if phi is None else 48 * np.log2(float(vo.ratio(phi)))


SIGNALS = {"vowel150": lambda: vowel(150.0, seed=1), "vowel200": lambda: vowel(200.0, seed=2), "speech": speech}


# ---- definition ---------------------------------------------------------------------------------------------------

def test_no_formant_is_the_pitch_shift():
    x = voiced_of(6000, 3)
    for s in (-5.0, 0.0, 7.0):
        assert np.array_equal(vo.voice_shift(x, s), po.pitch_shift(x, s))
        assert np.array_equal(vo.error_scale(x, s), po.error_scale(x, s))


@pytest.mark.parametrize("n", [0, 1, 300, 512, 513, 9000])
def test_copy_rows(n):
    x = signal_of(max(n, 1), 3)[:n]
    assert np.array_equal(vo.voice_shift(x, 0.0, 0.0), x.astype(np.float64))
    assert np.array_equal(vo.voice_shift(x, -0.0, -0.0), x.astype(np.float64))
    if n <= do.PAD:
        assert np.array_equal(vo.voice_shift(x, 5.0, 3.0), x.astype(np.float64))
    else:
        assert not np.array_equal(vo.voice_shift(x, 0.0, 3.0), x.astype(np.float64))   # s = 0, phi != 0 is filtered


def test_unmoved_formants_at_zero_shift_return_the_input():
    """s = 0, phi = 0 forced through the vocoder: u = t gives g = 1 and psi = 0, so the STFT round trip returns x"""
    x = voiced_of(9000, 4)
    y = vo.voice_shift(x, 0.0, 0.0, force=True)
    assert np.abs(y - x).max() <= 1e-9


def test_silence_gives_unit_gain():
    E = vo.envelope(np.zeros(do.N_BINS))
    k = np.arange(do.N_BINS)
    for phi in (-12.0, -3.0, 4.0, 12.0):
        g = vo.gains(E, k, k, vo.ratio(phi))
        assert np.abs(g - 1).max() <= 1e-12, phi
    x = np.zeros(4000, np.float32)
    assert np.array_equal(vo.voice_shift(x, 0.0, 5.0), np.zeros(4000))


def test_envelope_is_the_liftered_cepstrum():
    """E equals the order-26 lifter of the real cepstrum computed by an FFT of the even extension"""
    a = np.abs(do.stft(voiced_of(4000, 2)))[5]
    E = vo.envelope(a)
    m = a.max()
    l = np.log(np.maximum(a, 1e-4 * m))
    cep = np.fft.irfft(l, do.N_FFT)
    cep[vo.Q + 1: do.N_FFT - vo.Q] = 0
    assert np.abs(np.fft.rfft(cep).real - E).max() <= 1e-9


def test_gain_caps_the_boost_only():
    E = np.zeros(do.N_BINS)
    E[50] = -10.0                                 # a deep notch at bin 50's source: its boost is capped at +24 dB
    E[300] = -10.0                                # a deep notch where bin 150 reads (u = 300): attenuated in full
    g = vo.gains(E, np.array([50, 150]), np.array([50, 150]), vo.ratio(-12.0))
    assert g[0] == pytest.approx(10 ** (24 / 20)) and g[1] == pytest.approx(np.exp(-10.0))
    assert vo.gains(E, np.array([300]), np.array([300]), 1.0)[0] == 1.0
    assert vo.envelope_at(np.arange(513.0), 600.0) == 512.0 and vo.envelope_at(np.arange(513.0), 10.25) == 10.25


# ---- it does what it says -----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def oracle_warps():
    out = {}
    for name, sig in SIGNALS.items():
        x = sig()
        for s, phi in KEEP_MOVE + LEGACY:
            y = vo.voice_shift(x, s, phi)
            out[name, s, phi] = (warp_steps(x, y), f0_of(y[SR // 4: 3 * SR // 4]) if name != "speech" else None,
                                 f0_of(x[SR // 4: 3 * SR // 4]) if name != "speech" else None)
    return out


@pytest.mark.parametrize("name", list(SIGNALS))
def test_envelope_warp_is_f_and_pitch_is_r(oracle_warps, name):
    for s, phi in KEEP_MOVE + LEGACY:
        j, f0y, f0x = oracle_warps[name, s, phi]
        want = expected_steps(s, phi)
        print(f"{name} s={s} phi={phi}: warp {j} steps, expected {want:.2f}")
        assert abs(j - want) <= (1 if phi is None else 4), (name, s, phi, j, want)
        if f0y is not None:
            assert abs(f0y / (float(po.ratio(s)) * f0x) - 1) <= 0.02, (name, s, phi, f0y, f0x)


# ---- fp32 emulation and the tolerance -------------------------------------------------------------------------

def f32(v):
    return np.asarray(v, np.float64).astype(np.float32)


def fma32(a, b, c):
    """fmaf in fp32: the exact product (48 bits fit a double) plus c, rounded once more"""
    return f32(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64))


COS32 = f32(np.cos(2 * np.pi * np.arange(do.N_FFT) / do.N_FFT))     # the twiddle table's real parts


def emulate_envelope(a32):
    """E [F, 513] in fp32 in the kernel's order: lane segments of 16 bins (lane 31 also 512) in ascending order, an
    xor-shuffle tree over the lanes, fmaf sums over q ascending"""
    F = a32.shape[0]
    m = a32.max(axis=1, keepdims=True)
    lo = np.maximum(f32(np.float32(1e-4) * m), np.float32(1e-30))
    l = f32(np.log(np.maximum(a32, lo).astype(np.float64)))
    k = np.arange(do.N_BINS)
    wl = np.where((k == 0) | (k == do.N_BINS - 1), l, f32(2 * l.astype(np.float64)))
    seg = np.zeros((F, 32, 17), np.float32)
    kk = np.full((32, 17), -1)
    for lane in range(32):
        cnt = 17 if lane == 31 else 16
        seg[:, lane, :cnt] = wl[:, 16 * lane: 16 * lane + cnt]
        kk[lane, :cnt] = np.arange(16 * lane, 16 * lane + cnt)
    c = np.zeros((F, vo.Q + 1), np.float32)
    for q in range(vo.Q + 1):
        p = np.zeros((F, 32), np.float32)
        for i in range(17):
            cs = np.where(kk[:, i] >= 0, COS32[(np.maximum(kk[:, i], 0) * q) % do.N_FFT], 0).astype(np.float32)
            p = np.where(kk[None, :, i] >= 0, fma32(seg[:, :, i], cs[None, :], p), p)
        for d in (16, 8, 4, 2, 1):
            p = f32(p.astype(np.float64) + p[:, np.arange(32) ^ d])
        c[:, q] = p[:, 0] * np.float32(1.0 / do.N_FFT)
    s = np.zeros((F, do.N_BINS), np.float32)
    for q in range(1, vo.Q + 1):
        s = fma32(c[:, q: q + 1], COS32[(k * q) % do.N_FFT][None, :], s)
    return f32(c[:, :1].astype(np.float64) + 2 * s.astype(np.float64))


def emulate_gains(E, k, t, f):
    u = t.astype(np.float64) / float(np.float32(f))
    i = np.minimum(np.floor(u), do.N_BINS - 1).astype(np.int64)
    j = np.minimum(i + 1, do.N_BINS - 1)
    fr = f32(u - i)
    e0 = E[i]
    eu = np.where(u >= do.N_BINS - 1, E[do.N_BINS - 1], fma32(fr, f32(E[j].astype(np.float64) - e0), e0))
    d = np.minimum(f32(eu.astype(np.float64) - E[k]), np.float32(vo.CAP))
    return f32(np.exp(d.astype(np.float64)))


def emulate(x, s, phi, dec, bf16=False):
    """the kernels' arithmetic in fp32 under the decisions `dec` (test_pitch_cpu.emulate with the envelope and the gain);
    `bf16` rounds the spectra to bf16"""
    x = np.asarray(x, np.float32)
    n = x.size
    r = float(po.ratio(s))
    f = float(vo.ratio(phi))
    w = do.window().astype(np.float32)
    F = do.n_frames(n)
    xp = np.pad(x, do.PAD + 1, mode="reflect")
    idx = do.HOP * np.arange(F)[:, None] + np.arange(do.N_FFT)[None, :] + 1
    X = torch.fft.fft(torch.from_numpy(xp[idx] * w).to(torch.complex64), dim=1)[:, : do.N_BINS]
    re, im = X.real.numpy(), X.imag.numpy()
    if bf16:
        re, im = to_bf16(re), to_bf16(im)
    a32 = f32(np.sqrt(fma32(re, re, f32(im.astype(np.float64) * im))))
    E = emulate_envelope(a32)
    th = np.arctan2(im.astype(np.float64), re.astype(np.float64))
    k = np.arange(do.N_BINS)
    Z = np.zeros((F, do.N_BINS), np.complex64)
    psi_prev = np.zeros(do.N_BINS)
    for t in range(F):
        flags = (dec[t] & 1) == 1
        own = po.owners(flags)
        pk = np.flatnonzero(flags)
        om = 2 * np.pi * pk / do.N_FFT
        prev = np.zeros(pk.size)
        if t > 0:
            d = th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * do.HOP / do.N_FFT
            om = om + po.deviation(d, (dec[t][pk] >> 1 & 1) == 1) / do.HOP
            prev = psi_prev[pk]
        psi_of = np.zeros(do.N_BINS)
        psi_of[pk] = po.princarg(prev + do.HOP * (r - 1) * om)
        has = own >= 0
        psi = np.where(has, psi_of[np.maximum(own, 0)], 0.0)
        D = np.where(has, np.rint((r - 1) * own), 0).astype(np.int64)
        j = k + D
        ok = has & (j >= 0) & (j < do.N_BINS)
        c, sn = np.cos(psi).astype(np.float32), np.sin(psi).astype(np.float32)
        zr = (re[t] * c - im[t] * sn).astype(np.float32)
        zi = (re[t] * sn + im[t] * c).astype(np.float32)
        g = np.ones(do.N_BINS, np.float32)
        g[ok] = emulate_gains(E[t], k[ok], j[ok], f)
        zr, zi = zr * g, zi * g
        sign = np.where(D % 2 == 1, np.float32(-1), np.float32(1))
        np.add.at(Z[t], j[ok], ((zr + 1j * zi) * sign).astype(np.complex64)[ok])
        psi_prev = psi
    Zt = torch.from_numpy(Z)
    full = torch.cat([Zt, torch.conj(Zt[:, 1: do.N_BINS - 1]).flip(1)], dim=1)
    yf = (torch.fft.fft(torch.conj(full), dim=1).real.numpy() * np.float32(1.0 / do.N_FFT)) * w
    acc = np.zeros(do.N_FFT + do.HOP * (F - 1), np.float32)
    env = np.zeros_like(acc)
    w2 = w.astype(np.float64) ** 2
    for fi in range(F):
        sl = slice(do.HOP * fi, do.HOP * fi + do.N_FFT)
        acc[sl] = acc[sl] + yf[fi]
        env[sl] = (w2 + env[sl].astype(np.float64)).astype(np.float32)
    return acc[do.PAD: do.PAD + n] / env[do.PAD: do.PAD + n]


def test_bound_has_headroom_over_the_emulation():
    """TOL_F is at least 4x the worst fp32 emulation of the kernels (under float64's decisions) over s in {-12, -5, 0,
    3, 12} x phi in {-5, 0, 4} on the pitch shifter's test rows, and at least 5x below what spectra rounded to bf16
    give"""
    worst, worst_bf = 0.0, np.inf
    for n, sig in ((1025, voiced_of), (3001, signal_of), (24000, voiced_of), (24000, signal_of)):
        x = sig(n, n + 1)
        for s in (-12.0, -5.0, 0.0, 3.0, 12.0):
            for phi in (-5.0, 0.0, 4.0):
                if s == 0.0 and phi == 0.0:
                    continue                                   # a copy
                dec = po.decisions_of(x, s if s != 0.0 else 1.0)     # at r = 1 only the peak flags count, not the sides
                y64 = vo.voice_shift(x, s, phi, decisions=dec)
                scale = vo.error_scale(x, s, phi)
                worst = max(worst, float((np.abs(emulate(x, s, phi, dec) - y64) / scale).max()))
                if n == 24000:
                    worst_bf = min(worst_bf, float((np.abs(emulate(x, s, phi, dec, bf16=True) - y64) / scale).max()))
    print(f"fp32 emulation {worst:.2e}, bf16 spectra {worst_bf:.2e} (TOL_F {TOL_F:.0e})")
    assert 4 * worst <= TOL_F, worst
    assert worst_bf >= 5 * TOL_F, worst_bf


# ---- the Python layer against a recording library -------------------------------------------------------------------

class _Lib:
    def __init__(self):
        self.calls = []
        self.arrays = {}

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, [self.arrays.get(a, a) if isinstance(a, int) else a for a in args]))
            if name.endswith("_create"):
                for a in args:
                    if type(a).__name__ == "CArgObject":
                        a._obj.value = 0x1234 if isinstance(a._obj, C.c_void_p) else 40
            return 0
        return fn


@pytest.fixture
def eng(monkeypatch):
    from viettts_b200 import engine as E
    lib = _Lib()

    def ptr(a):
        if a is None:
            return None
        addr = a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr()
        lib.arrays[addr] = a.copy() if isinstance(a, np.ndarray) else a
        return addr
    monkeypatch.setattr(E, "_ptr", ptr)
    e = E.Engine.__new__(E.Engine)
    e.lib, e.h, e.device = lib, C.c_void_p(99), 0
    return e


def test_one_shot_calls_pick_the_entry_point(eng):
    x = np.zeros((2, 700), np.float32)
    eng.pitch_shift(x, [3.0, -2.0])
    eng.pitch_shift(x, [3.0, -2.0], formant=0.0)
    eng.pitch_shift(x, 0.0, formant=[1.5, -4.0])
    names = [n for n, _ in eng.lib.calls]
    assert names == ["vtts_pitch_shift_host", "vtts_voice_shift_host", "vtts_voice_shift_host"]
    assert list(eng.lib.calls[1][1][6]) == [0.0, 0.0] and list(eng.lib.calls[2][1][6]) == [1.5, -4.0]
    for bad in (np.nan, np.inf, 12.5, -13.0, [1.0, 2.0, 3.0]):
        with pytest.raises(ValueError):
            eng.pitch_shift(x, 0.0, formant=bad)
    assert len(eng.lib.calls) == 3


def test_voice_stream_marshalling_and_carry(eng):
    from viettts_b200 import engine as E
    st = E.VoiceShiftStream(eng, 3, 20)
    x = np.zeros((3, 20), np.float32)
    st.push(x, [1, 1, 0], begin=[True, True, False], semitones=[3.0, -2.0, 5.0])             # both slots follow the pitch
    st.push(x, [1, 1, 1], begin=[False, False, True], semitones=7.0, formant=-3.0)
    st.push(x, [1, 0, 1], begin=[True, False, False], semitones=[1.0, 9.0, 9.0], formant=[2.0, 9.0, 9.0])
    pushes = [r for n, r in eng.lib.calls if n == "vtts_voice_shift_stream_push_host"]
    assert len(pushes) == 3 and pushes[0][6] is None
    f1, f2 = pushes[1][6], pushes[2][6]
    assert np.isnan(f1[:2]).all() and f1[2] == -3.0
    assert f2[0] == 2.0 and np.isnan(f2[1]) and f2[2] == -3.0
    assert list(st.shift) == [1.0, -2.0, 7.0] and st.formant[0] == 2.0 and np.isnan(st.formant[1]) and st.formant[2] == -3.0
    assert [n for n, _ in eng.lib.calls if "push" in n] == ["vtts_voice_shift_stream_push_host"] * 3
    st.close()
    assert eng.lib.calls[-1][0] == "vtts_pitch_shift_stream_destroy"


def test_chain_and_cli_take_the_formant(monkeypatch, tmp_path):
    from viettts_b200 import engine as E
    from viettts_b200 import synthesizer
    ch = E.AudioChain(formant=0.0)
    assert [s[0] for s in ch._stages()] == ["ps"] and ch.semitones is None and ch.formant == 0.0
    with pytest.raises(E.OptionError):
        E.AudioChain(semitones=2.0, formant=13.0)

    class Rec:
        def __init__(self):
            self.calls = []

        def pitch_shift(self, w, s, formant=None):
            self.calls.append((s, formant))
            return w
    rec = Rec()
    E.AudioChain(semitones=4.0, formant=0.0).run(rec, np.zeros(10, np.float32))
    E.AudioChain(formant=-3.0).run(rec, np.zeros(10, np.float32))
    E.AudioChain(semitones=2.0).run(rec, np.zeros(10, np.float32))
    assert rec.calls == [(4.0, 0.0), (0.0, -3.0), (2.0, None)]
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", "--formant", "20"])
