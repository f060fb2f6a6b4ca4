"""CPU: the pitch shifter's definition (oracle/pitch_oracle.py), its stream schedule and the tolerance the GPU tests hold
it to.

The oracle is checked on what a pitch shift must do: tones land on f * r with their energy around it, a harmonic series
stays harmonic, a glide keeps its level (and a variant without the frame-centre sign does not), a tone pushed past
Nyquist is dropped, s = 0 and short rows are copies.  TOL -- the bound |y - y64| <= TOL * pitch_oracle.error_scale per
output -- comes from an fp32 emulation of the kernels run under float64's decisions, as test_denoise_cpu.py derives
the denoiser's."""
import numpy as np
import pytest
import torch

from oracle import denoise_oracle as do
from oracle import pitch_oracle as po
from test_denoise_cpu import signal_of

SR = 16000
SHIFTS = [-12.0, -5.0, 3.0, 7.0, 12.0]
TOL = 2e-5    # per output, relative to error_scale (see test_bound_has_headroom_over_the_emulation)
DEC_MARGIN = 1e-5   # device decisions may differ from float64's only where float64's margin is below this x the frame norm


def tone(f, n=SR, amp=0.5):
    return amp * np.sin(2 * np.pi * f * np.arange(n) / SR)


def interior(y, cut=2000):
    return y[cut:-cut]


def peak_freq(y):
    """frequency of the largest peak of a 16x zero-padded Hann spectrum, refined by a parabola through the log magnitudes"""
    w = np.hanning(y.size)
    Y = np.abs(np.fft.rfft(y * w, 16 * y.size))
    i = int(np.argmax(Y))
    a, b, c = np.log(Y[i - 1: i + 2])
    d = 0.5 * (a - c) / (a - 2 * b + c)
    return (i + d) * SR / (16 * y.size)


def energy_near(y, freqs, width):
    Y = np.abs(np.fft.rfft(y * np.hanning(y.size))) ** 2
    fr = np.fft.rfftfreq(y.size, 1 / SR)
    near = np.zeros(fr.size, bool)
    for f in np.atleast_1d(freqs):
        near |= np.abs(fr - f) < width
    return Y[near].sum() / Y.sum()


# ---- definition ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [0, 1, 300, 512, 513, 1025, 9000])
def test_zero_shift_and_short_rows_are_copies(n):
    x = signal_of(max(n, 1), 3)[:n]
    assert np.array_equal(po.pitch_shift(x, 0.0), x.astype(np.float64))
    assert np.array_equal(po.pitch_shift(x, -0.0), x.astype(np.float64))
    if n <= do.PAD:
        assert np.array_equal(po.pitch_shift(x, 7.0), x.astype(np.float64))


def test_ratio_is_fp32_of_the_double_power():
    assert po.ratio(12) == np.float32(2.0) and po.ratio(-12) == np.float32(0.5) and po.ratio(0) == np.float32(1.0)
    assert po.ratio(3) == np.float32(2.0 ** 0.25)
    for bad in (12.5, -13, np.nan, np.inf):
        with pytest.raises(ValueError):
            po.ratio(bad)


def test_owners_take_the_nearest_peak_and_the_lower_one_on_a_tie():
    flags = np.zeros(513, bool)
    flags[[10, 14, 100]] = True
    own = po.owners(flags)
    assert list(own[:13]) == [10] * 13                    # 12 is 2 from both 10 and 14: the lower
    assert list(own[13:58]) == [14] * 45 and own[57] == 14 and own[58] == 100 and np.all(own[58:] == 100)
    assert np.all(po.owners(np.zeros(513, bool)) == -1)
    a = np.zeros(513)
    a[[0, 5, 6, 512]] = [2.0, 1.0, 1.0, 3.0]
    assert list(np.flatnonzero(po.peak_flags(a))) == [0, 5, 512]       # a plateau's first bin, the edges against -1


@pytest.mark.parametrize("f", [100.0, 250.0, 440.0, 1000.0, 3000.0])
@pytest.mark.parametrize("s", SHIFTS)
def test_tones_land_on_the_shifted_frequency(f, s):
    target = f * float(po.ratio(s))
    assert 50.0 <= target <= 6000.0
    y = interior(po.pitch_shift(tone(f), s))
    assert abs(peak_freq(y) - target) <= 0.1, (f, s, peak_freq(y), target)
    assert energy_near(y, target, 15.0) >= 0.999, (f, s, energy_near(y, target, 15.0))


def test_harmonic_series_stays_harmonic():
    t = np.arange(SR) / SR
    x = sum(0.2 / h * np.sin(2 * np.pi * 150 * h * t + h) for h in range(1, 20))
    y = interior(po.pitch_shift(x, 4.0))
    r = float(po.ratio(4.0))
    assert energy_near(y, [150 * r * h for h in range(1, 30)], 10.0) >= 0.999


def rms_envelope(y):
    return np.sqrt(np.convolve(y ** 2, np.ones(256) / 256, "valid"))


def test_glide_keeps_its_level_only_with_the_frame_centre_sign():
    t = np.arange(2 * SR) / SR
    x = 0.5 * np.sin(2 * np.pi * (200 * t + 100 * t ** 2))          # 200 -> 600 Hz
    env = rms_envelope(interior(po.pitch_shift(x, 3.0)))
    bad = rms_envelope(interior(po.pitch_shift(x, 3.0, frame_centre=False)))
    print(f"glide RMS min / max {env.min() / env.max():.3f}, without (-1)^D {bad.min() / bad.max():.3f}")
    assert env.min() / env.max() >= 0.8
    assert bad.min() / bad.max() < 0.8


def test_tone_past_nyquist_is_dropped():
    x = tone(5000.0)
    y = po.pitch_shift(x, 12.0)                                         # 10 kHz > 8 kHz
    assert (interior(y) ** 2).sum() <= 1e-12 * (interior(x) ** 2).sum()


# ---- stream schedule ------------------------------------------------------------------------------------------

def test_stream_schedule_is_the_denoisers_and_equals_counting():
    assert po.emitted_closed_form is do.emitted_closed_form and po.schedule is do.schedule and po.LOOKAHEAD == 1023
    for P in range(0, 5001):
        assert po.emitted_closed_form(P) == po.emitted(P), P
    assert po.lookahead() == po.LOOKAHEAD


def frames_final(P: int, end: bool) -> int:
    """frames a stream slot has scanned after P inputs: those that read no input past P - 1 (frame 0 reflects sample
    512 into its first half, so it needs P > 512), every frame with END"""
    if end:
        return do.n_frames(P) if P > do.PAD else 0
    return (P - do.PAD) // do.HOP + 1 if P > do.PAD else 0


def test_scanned_frames_cover_every_emitted_output():
    """each output a slot emits reads only frames it has scanned, and every scanned frame reads only inputs it has"""
    for P in range(0, 4000):
        q = frames_final(P, False)
        e = po.emitted_closed_form(P)
        if e:
            assert (e - 1 + do.PAD) // do.HOP < q, P          # the last frame covering output e - 1
        if q:
            g = q - 1
            assert do.HOP * g + do.PAD - 1 <= P - 1 and (g > 0 or P - 1 >= do.PAD), P


# ---- fp32 emulation and the tolerance -----------------------------------------------------------------------

def emulate(x, s, dec, shift=0, bf16=False):
    """the kernels' arithmetic in fp32 under the decisions `dec`: windowed frame, complex64 FFT, theta = atan2 in double
    of the fp32 bins, the double phase recurrence, e^(i psi) rounded to fp32, the fp32 rotation and sums in ascending k,
    the inverse of the Hermitian spectrum times 1 / 1024 times w, overlap-add in ascending frame order over an fp32
    envelope.  Variants: frames taken `shift` samples late, spectra rounded to bf16."""
    from test_denoise_cpu import to_bf16
    x = np.asarray(x, np.float32)
    n = x.size
    r = float(po.ratio(s))
    w = do.window().astype(np.float32)
    F = do.n_frames(n)
    xp = np.pad(x, do.PAD + 1, mode="reflect")
    idx = do.HOP * np.arange(F)[:, None] + np.arange(do.N_FFT)[None, :] + 1 + shift
    X = torch.fft.fft(torch.from_numpy(xp[idx] * w).to(torch.complex64), dim=1)[:, : do.N_BINS]
    re, im = X.real.numpy(), X.imag.numpy()
    if bf16:
        re, im = to_bf16(re), to_bf16(im)
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
        sign = np.where(D % 2 == 1, np.float32(-1), np.float32(1))
        np.add.at(Z[t], j[ok], ((zr + 1j * zi) * sign).astype(np.complex64)[ok])
        psi_prev = psi
    Zt = torch.from_numpy(Z)
    full = torch.cat([Zt, torch.conj(Zt[:, 1: do.N_BINS - 1]).flip(1)], dim=1)
    yf = (torch.fft.fft(torch.conj(full), dim=1).real.numpy() * np.float32(1.0 / do.N_FFT)) * w
    acc = np.zeros(do.N_FFT + do.HOP * (F - 1), np.float32)
    env = np.zeros_like(acc)
    w2 = w.astype(np.float64) ** 2
    for f in range(F):
        sl = slice(do.HOP * f, do.HOP * f + do.N_FFT)
        acc[sl] = acc[sl] + yf[f]
        env[sl] = (w2 + env[sl].astype(np.float64)).astype(np.float32)
    return acc[do.PAD: do.PAD + n] / env[do.PAD: do.PAD + n]


def voiced_of(n, seed=0):
    """a voiced test row: a harmonic series on a gliding pitch with noise, a faint stretch, then a louder burst"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    ph = 2 * np.pi * (140 * t + 30 * t ** 2)
    x = sum(0.3 / h * np.sin(h * ph + h) for h in range(1, 12)) + 0.02 * rng.standard_normal(n)
    x[n // 3: n // 2] *= 1e-2
    return x.astype(np.float32)


def test_bound_has_headroom_over_the_emulation():
    """TOL is at least 4x the worst fp32 emulation of the kernels (under float64's decisions), at least 5x below what
    spectra rounded to bf16 would give and at least 10x below frames shifted by one sample.  The emulation's error is
    ~2e-7 on most rows; its tail comes from weak peaks, whose fp32 phase error their region's stronger bins carry."""
    worst, worst_bf, worst_shift = 0.0, np.inf, np.inf
    for n, sig in ((513, signal_of), (1025, voiced_of), (3001, signal_of), (24000, voiced_of), (24000, signal_of)):
        x = sig(n, n + 1)
        for s in (-12.0, -5.0, 3.0, 12.0):
            dec = po.decisions_of(x, s)
            y64 = po.pitch_shift(x, s, decisions=dec)
            scale = po.error_scale(x, s)
            worst = max(worst, float((np.abs(emulate(x, s, dec) - y64) / scale).max()))
            if n == 24000:
                worst_bf = min(worst_bf, float((np.abs(emulate(x, s, dec, bf16=True) - y64) / scale).max()))
                worst_shift = min(worst_shift, float((np.abs(emulate(x, s, dec, shift=1) - y64) / scale).max()))
    print(f"fp32 emulation {worst:.2e}, bf16 spectra {worst_bf:.2e}, frames shifted by one {worst_shift:.2e} (TOL {TOL:.0e})")
    assert 4 * worst <= TOL, worst
    assert worst_bf >= 5 * TOL, worst_bf
    assert worst_shift >= 10 * TOL, worst_shift


def decision_margins(x, dec):
    """per frame and bin, float64's margin of each decision the device took, over the frame's L2 norm ||w x_f||: for a
    peak flag the smallest |a[k] - a[k -/+ 1]| (or a[k]) it compares, for a branch the distance of the deviation from
    the cut at +-pi times the smaller magnitude of the two frames at that bin (the phase error of an fp32 bin is its
    error over its magnitude)"""
    x = np.asarray(x, np.float64)
    _, a, th = po.analysis(x)
    norm = np.linalg.norm(do.frames(x) * do.window(), axis=1)[:, None]
    ap = np.concatenate([np.full((a.shape[0], 1), -1.0), a, np.full((a.shape[0], 1), -1.0)], axis=1)
    flag_margin = np.minimum(np.minimum(np.abs(a - ap[:, :-2]), np.abs(a - ap[:, 2:])), a) / norm
    k = np.arange(do.N_BINS)
    d = th[1:] - th[:-1] - 2 * np.pi * k * do.HOP / do.N_FFT
    branch = np.zeros_like(a)
    branch[1:] = (np.pi - np.abs(po.deviation(d))) * np.minimum(a[1:], a[:-1]) / np.maximum(norm[1:], norm[:-1])
    branch[0] = np.inf
    return flag_margin, branch


def test_emulated_decisions_differ_only_at_small_margins():
    """the fp32 spectra's own decisions differ from float64's only where float64's margin is below DEC_MARGIN: the
    criterion the GPU test applies to the device"""
    x = voiced_of(24000, 5)
    xf = x.astype(np.float32)
    F = do.n_frames(x.size)
    xp = np.pad(xf, do.PAD, mode="reflect")
    idx = do.HOP * np.arange(F)[:, None] + np.arange(do.N_FFT)[None, :]
    X = torch.fft.fft(torch.from_numpy(xp[idx] * do.window().astype(np.float32)).to(torch.complex64), dim=1)[:, : do.N_BINS].numpy()
    a32 = np.sqrt(X.real * X.real + X.imag * X.imag)
    th32 = np.arctan2(X.imag.astype(np.float64), X.real.astype(np.float64))
    dec64 = po.decisions_of(x, 3.0)
    flag_m, branch_m = decision_margins(x, dec64)
    fl32 = np.stack([po.peak_flags(a) for a in a32])
    fl64 = (dec64 & 1) == 1
    assert np.all(flag_m[fl32 != fl64] < DEC_MARGIN)
    k = np.arange(do.N_BINS)
    neg32 = po.deviation(th32[1:] - th32[:-1] - 2 * np.pi * k * do.HOP / do.N_FFT) < 0
    both = fl32[1:] & fl64[1:]
    diff = both & (neg32 != ((dec64[1:] >> 1 & 1) == 1))
    assert np.all(branch_m[1:][diff] < DEC_MARGIN)
    print(f"flag flips {int((fl32 != fl64).sum())}, branch flips {int(diff.sum())} of {int(fl64.sum())} peaks")
