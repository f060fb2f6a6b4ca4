"""CPU: the time stretcher's definition (oracle/time_stretch_oracle.py: time_stretch, the pitch shifter's vocoder with
moving analysis frames), its stream schedule and the tolerance the GPU tests hold it to.

The shared vocoder routine must state the pitch shifter exactly as oracle/pitch_oracle.py does; the two are compared
bit for bit.  TOL -- the bound |y - y64| <= TOL *
time_stretch_oracle.stretch_error_scale per output -- comes from an fp32 emulation of the kernels run under float64's
decisions, as test_pitch_cpu.py derives the pitch shifter's."""
import numpy as np
import pytest
import torch

from oracle import denoise_oracle as do
from oracle import pitch_oracle as po
from oracle import time_stretch_oracle as tso
from test_denoise_cpu import signal_of
from test_pitch_cpu import voiced_of

SR = 16000
TEMPOS = [0.5, 0.75, 1.25, 1.6180339, 2.0]
TOL = 1.2e-4        # per output, relative to stretch_error_scale (see test_bound_has_headroom_over_the_emulation)
DEC_MARGIN = 1e-5   # device decisions may differ from float64's only where float64's margin is below this x the frame norm
LEVEL_DB = 0.1      # a stationary tone's steady-state level after the stretch, within this many dB of the input's


# ---- definition ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,s", [(513, 3.0), (1025, -12.0), (3001, 7.5), (9000, 12.0), (24000, -5.0), (24000, 0.5)])
def test_pitch_shift_is_the_shared_routine_at_tempo_one(n, s):
    """the shared vocoder at a_t = 256 t and ratio r is the pitch shifter's statement, bits and decisions alike"""
    x = (voiced_of if n % 2 else signal_of)(n, n + 3)
    assert np.array_equal(tso.pitch_shift(x, s), po.pitch_shift(x, s))
    assert np.array_equal(tso.decisions_of(x, s), po.decisions_of(x, s))


@pytest.mark.parametrize("n", [0, 1, 300, 512, 513, 1025, 9000])
def test_unit_tempo_and_short_rows_are_copies(n):
    x = signal_of(max(n, 1), 3)[:n].astype(np.float64)
    assert np.array_equal(tso.time_stretch(x, 1.0), x)
    if n <= do.PAD:
        for a in TEMPOS:
            M = tso.stretch_length(n, a)
            y = tso.time_stretch(x, a)
            k = min(n, M)
            assert y.shape == (M,) and np.array_equal(y[:k], x[:k]) and not y[k:].any(), (n, a)


@pytest.mark.parametrize("n", [0, 1, 512, 513, 1023, 1025, 80128])
@pytest.mark.parametrize("a", [0.5, 0.75, 1.0, 1.25, 2.0, 1.3333334])
def test_output_length(n, a):
    M = int(np.floor(n / float(np.float32(a)) + 0.5))
    assert tso.stretch_length(n, a) == M
    x = signal_of(max(n, 1), 5)[:n]
    assert tso.time_stretch(x, a).shape == (M,)
    assert tso.stretch_centres(n, a).size == M // do.HOP + 1


def test_tempo_is_checked():
    assert tso.tempo_of(2) == 2.0 and tso.tempo_of(0.5) == 0.5
    for bad in (0.49, 2.01, np.nan, np.inf, 0.0, -1.0):
        with pytest.raises(ValueError):
            tso.tempo_of(bad)


def test_hops_are_at_least_one():
    """h_t = a_t - a_t-1 >= 1 for every row: the clamp at n - 1 reaches the last frame only (tso.hops asserts it)"""
    for a in TEMPOS + [0.5000001, 1.9999999, 1.001, 0.999]:
        for n in list(range(513, 3000, 7)) + [80128, 80128 + 255]:
            h = tso.hops(tso.stretch_centres(n, a))
            assert h.min() >= 1, (a, n)


def peak_bin(y):
    Y = np.abs(np.fft.rfft(y * np.hanning(y.size)))
    return int(np.argmax(Y)), SR / y.size


@pytest.mark.parametrize("f", [150.0, 440.0, 1000.0, 3000.0])
@pytest.mark.parametrize("a", TEMPOS)
def test_stationary_tone_keeps_its_frequency_and_level(f, a):
    x = 0.5 * np.sin(2 * np.pi * f * np.arange(SR) / SR)
    y = tso.time_stretch(x, a)[2000:-2000]
    i, df = peak_bin(y)
    assert abs(i * df - f) <= df, (f, a, i * df)
    db = 20 * np.log10(np.sqrt(np.mean(y ** 2)) / np.sqrt(np.mean(x[2000:-2000] ** 2)))
    assert abs(db) <= LEVEL_DB, (f, a, db)


# ---- stream schedule ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("a", [0.5, 0.75, 1.25, 1.37, 2.0])
def test_stream_schedule_is_tight(a):
    """a released output never depends on input past the ones received, and the first unreleased one does"""
    N = 7000
    x1 = voiced_of(N, 21).astype(np.float64)
    y1 = tso.time_stretch(x1, a)
    rng = np.random.default_rng(5)
    for P in (513, 700, 1024, 1500, 2345, 3001, 4096):
        E = tso.stretch_emitted(P, a)
        x2 = x1.copy()
        x2[P:] = 0.3 * rng.standard_normal(N - P)
        y2 = tso.time_stretch(x2, a)
        assert E <= y1.size
        assert np.array_equal(y1[:E], y2[:E]), (a, P, E)
        assert y1[E] != y2[E], (a, P, E)


@pytest.mark.parametrize("a", TEMPOS + [1.0])
def test_stream_schedule_reads_only_scanned_frames_and_received_inputs(a):
    """each frame scanned before END reads no input past P - 1 (and frame 0 needs P > 512), each released output reads
    only scanned frames, and the release lags P / alpha by less than the lookahead"""
    for P in range(0, 9000, 3):
        q = tso.stretch_scanned(P, a)
        e = tso.stretch_emitted(P, a)
        if q:
            assert P > do.PAD and int(np.rint(256.0 * (q - 1) * tso.tempo_of(a))) + do.PAD - 1 <= P - 1, (a, P)
        if e and tso.tempo_of(a) != 1.0:
            assert (e - 1 + do.PAD - 1) // do.HOP < q, (a, P)
        assert e > P / tso.tempo_of(a) - tso.TS_LOOKAHEAD, (a, P, e)


def test_schedule_releases_everything_at_end():
    for a in TEMPOS:
        for pushes in ([1000] * 7, [1] * 900, [5000, 0], [300]):
            out = tso.stretch_schedule(pushes, a)
            assert min(out) >= 0 and sum(out) == tso.stretch_length(sum(pushes), a), (a, pushes)


# ---- fp32 emulation and the tolerance -----------------------------------------------------------------------

def emulate(x, a, dec, shift=0, bf16=False):
    """the kernels' arithmetic in fp32 under the decisions `dec`, as test_pitch_cpu.emulate with the analysis frames at
    the time stretcher's centres and r = 1.  Variants: frames taken `shift` samples late, spectra rounded to bf16."""
    from test_denoise_cpu import to_bf16
    x = np.asarray(x, np.float32)
    n = x.size
    M = tso.stretch_length(n, a)
    c = tso.stretch_centres(n, a)
    h = tso.hops(c)
    w = do.window().astype(np.float32)
    T = c.size
    xp = np.pad(x, do.PAD + 1, mode="reflect")
    idx = c[:, None] + np.arange(do.N_FFT)[None, :] + 1 + shift
    X = torch.fft.fft(torch.from_numpy(xp[idx] * w).to(torch.complex64), dim=1)[:, : do.N_BINS]
    re, im = X.real.numpy(), X.imag.numpy()
    if bf16:
        re, im = to_bf16(re), to_bf16(im)
    th = np.arctan2(im.astype(np.float64), re.astype(np.float64))
    Z = np.zeros((T, do.N_BINS), np.complex64)
    psi_prev = np.zeros(do.N_BINS)
    for t in range(T):
        flags = (dec[t] & 1) == 1
        own = tso.owners(flags)
        pk = np.flatnonzero(flags)
        om = 2 * np.pi * pk / do.N_FFT
        prev = np.zeros(pk.size)
        if t > 0:
            d = th[t][pk] - th[t - 1][pk] - 2 * np.pi * pk * h[t] / do.N_FFT
            om = om + tso.deviation(d, (dec[t][pk] >> 1 & 1) == 1) / h[t]
            prev = psi_prev[pk]
        psi_of = np.zeros(do.N_BINS)
        psi_of[pk] = tso.princarg(prev + (do.HOP - h[t]) * om)
        has = own >= 0
        psi = np.where(has, psi_of[np.maximum(own, 0)], 0.0)
        cs, sn = np.cos(psi).astype(np.float32), np.sin(psi).astype(np.float32)
        zr = (re[t] * cs - im[t] * sn).astype(np.float32)
        zi = (re[t] * sn + im[t] * cs).astype(np.float32)
        Z[t] = np.where(has, zr + 1j * zi, 0).astype(np.complex64)
        psi_prev = psi
    Zt = torch.from_numpy(Z)
    full = torch.cat([Zt, torch.conj(Zt[:, 1: do.N_BINS - 1]).flip(1)], dim=1)
    yf = (torch.fft.fft(torch.conj(full), dim=1).real.numpy() * np.float32(1.0 / do.N_FFT)) * w
    acc = np.zeros(do.N_FFT + do.HOP * (T - 1), np.float32)
    env = np.zeros_like(acc)
    w2 = w.astype(np.float64) ** 2
    for f in range(T):
        sl = slice(do.HOP * f, do.HOP * f + do.N_FFT)
        acc[sl] = acc[sl] + yf[f]
        env[sl] = (w2 + env[sl].astype(np.float64)).astype(np.float32)
    return acc[do.PAD: do.PAD + M] / env[do.PAD: do.PAD + M]


def test_bound_has_headroom_over_the_emulation():
    """TOL is at least 4x the worst fp32 emulation of the kernels (under float64's decisions), below what spectra
    rounded to bf16 would give and at least 100x below frames shifted by one sample.  The emulation's error is below
    1e-6 on most rows; its tail (2.7e-5, one 3001-sample row at tempo 1.25) comes from a weak peak whose fp32 phase
    error the recurrence carries through the frames of its region.  That tail is why TOL is 6x the pitch shifter's."""
    worst, worst_bf, worst_shift = 0.0, np.inf, np.inf
    for n, sig in ((513, signal_of), (1025, voiced_of), (3001, signal_of), (24000, voiced_of), (24000, signal_of)):
        x = sig(n, n + 1)
        for a in (0.5, 0.75, 1.25, 2.0):
            dec = tso.stretch_decisions_of(x, a)
            y64 = tso.time_stretch(x, a, decisions=dec)
            scale = tso.stretch_error_scale(x, a)
            worst = max(worst, float((np.abs(emulate(x, a, dec) - y64) / scale).max()))
            if n == 24000:
                worst_bf = min(worst_bf, float((np.abs(emulate(x, a, dec, bf16=True) - y64) / scale).max()))
                worst_shift = min(worst_shift, float((np.abs(emulate(x, a, dec, shift=1) - y64) / scale).max()))
    print(f"fp32 emulation {worst:.2e}, bf16 spectra {worst_bf:.2e}, frames shifted by one {worst_shift:.2e} (TOL {TOL:.0e})")
    assert 4 * worst <= TOL, worst
    assert worst_bf >= TOL, worst_bf
    assert worst_shift >= 100 * TOL, worst_shift


def decision_margins(x, a):
    """per frame and bin, float64's margin of each decision of the time stretcher over the frame's L2 norm, as
    test_pitch_cpu.decision_margins with the analysis frames at the stretcher's centres and hops.  A deviation with
    |e| <= pi / 2 takes no branch decision (its margin is 0, either side is right): a tone on a bin centre gives e ~ 0
    at every hop, and the sign of that rounding residue changes nothing."""
    x = np.asarray(x, np.float64)
    c = tso.stretch_centres(x.size, a)
    h = tso.hops(c)
    _, mag, th = tso.analysis(x, c)
    norm = np.linalg.norm(tso.frames_at(x, c) * do.window(), axis=1)[:, None]
    ap = np.concatenate([np.full((mag.shape[0], 1), -1.0), mag, np.full((mag.shape[0], 1), -1.0)], axis=1)
    flag_margin = np.minimum(np.minimum(np.abs(mag - ap[:, :-2]), np.abs(mag - ap[:, 2:])), mag) / norm
    k = np.arange(do.N_BINS)
    d = th[1:] - th[:-1] - 2 * np.pi * k[None, :] * h[1:, None] / do.N_FFT
    branch = np.zeros_like(mag)
    # the side only decides anything where |e| > pi / 2 (there the oracle moves e by 2 pi); near e = 0 its sign is free
    e = np.abs(tso.deviation(d))
    branch[1:] = np.where(e > np.pi / 2, (np.pi - e) * np.minimum(mag[1:], mag[:-1]) / np.maximum(norm[1:], norm[:-1]), 0.0)
    branch[0] = np.inf
    return flag_margin, branch


def test_emulated_decisions_differ_only_at_small_margins():
    """the fp32 spectra's own decisions differ from float64's only where float64's margin is below DEC_MARGIN: the
    criterion the GPU test applies to the device"""
    for a in (0.75, 2.0):
        x = voiced_of(24000, 5)
        c = tso.stretch_centres(x.size, a)
        h = tso.hops(c)
        xp = np.pad(x.astype(np.float32), do.PAD, mode="reflect")
        fr = xp[c[:, None] + np.arange(do.N_FFT)[None, :]] * do.window().astype(np.float32)
        X = torch.fft.fft(torch.from_numpy(fr).to(torch.complex64), dim=1)[:, : do.N_BINS].numpy()
        a32 = np.sqrt(X.real * X.real + X.imag * X.imag)
        th32 = np.arctan2(X.imag.astype(np.float64), X.real.astype(np.float64))
        dec64 = tso.stretch_decisions_of(x, a)
        flag_m, branch_m = decision_margins(x, a)
        fl32 = np.stack([tso.peak_flags(v) for v in a32])
        fl64 = (dec64 & 1) == 1
        assert np.all(flag_m[fl32 != fl64] < DEC_MARGIN), a
        k = np.arange(do.N_BINS)
        neg32 = tso.deviation(th32[1:] - th32[:-1] - 2 * np.pi * k[None, :] * h[1:, None] / do.N_FFT) < 0
        both = fl32[1:] & fl64[1:]
        diff = both & (neg32 != ((dec64[1:] >> 1 & 1) == 1))
        assert np.all(branch_m[1:][diff] < DEC_MARGIN), a
        print(f"tempo {a}: flag flips {int((fl32 != fl64).sum())}, branch flips {int(diff.sum())} of {int(fl64.sum())} peaks")
