"""CPU: the bias denoiser's definition, its stream schedule and the tolerance the GPU tests hold it to.

The oracle (oracle/denoise_oracle.py) is pinned against float64 torch.stft / torch.istft of the same definition; the
stream's emission formula and lookahead against the oracle's counting; and TOL -- the bound
|y - y64| <= TOL * denoise_oracle.error_scale per output -- against an fp32 emulation of the kernels (fp32 torch FFTs,
the kernels' order of operations), and against two wrong variants it must reject."""
import numpy as np
import pytest
import torch

from oracle import denoise_oracle as do

SR = 16000
LENGTHS = [513, 767, 768, 1023, 1024, 1025, 80128]
STRENGTHS = [0.0, 0.01, 0.1, 1.0]
TOL = 2e-7    # per output, relative to error_scale (see test_bound_has_headroom_over_the_emulation)


def signal_of(n, seed=0):
    """speech-like test row: a tone with noise, a silent stretch holding only a faint hiss, then a louder burst"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    x = 0.5 * np.sin(2 * np.pi * 220 * t) + 0.2 * rng.standard_normal(n)
    x[n // 3: 2 * n // 3] = 2e-3 * rng.standard_normal(2 * n // 3 - n // 3)
    return x.astype(np.float32)


def hiss_bias(seed=1):
    """a bias spectrum of the size a generator's hiss has: |X_0| of faint noise"""
    rng = np.random.default_rng(seed)
    return do.bias_of(3e-3 * rng.standard_normal(4096)).astype(np.float32)


def torch_reference(x, s, bias):
    """the definition through float64 torch.stft / torch.istft"""
    x = torch.from_numpy(np.asarray(x, np.float64))
    w = torch.hann_window(do.N_FFT, periodic=True, dtype=torch.float64)
    X = torch.stft(x, do.N_FFT, do.HOP, window=w, center=True, pad_mode="reflect", return_complex=True)   # [513, F]
    mag = X.abs()
    keep = torch.clamp(mag - s * torch.from_numpy(np.asarray(bias, np.float64))[:, None], min=0.0)
    gain = torch.where(mag > 0, keep / torch.where(mag > 0, mag, torch.ones_like(mag)), torch.zeros_like(mag))
    return torch.istft(X * gain, do.N_FFT, do.HOP, window=w, center=True, length=x.numel()).numpy()


def to_bf16(a):
    u = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return u.view(np.float32)


def emulate(x, s, bias, bf16_spectra=False, shift=0):
    """the kernels' arithmetic in fp32: windowed frame, forward FFT (complex64), |X|, M' = max(|X| - fp32(s) * beta, 0),
    gain M' / |X|, inverse FFT of the Hermitian spectrum, real part times 1 / 1024 times w; overlap-add in ascending
    frame order and an fp32 envelope of fused w * w + env steps, one division.  Variants: spectra rounded to bf16, and
    frames taken `shift` samples late."""
    x = np.asarray(x, np.float32)
    n = x.size
    if n <= do.PAD:
        return x.copy()
    w = do.window().astype(np.float32)
    F = do.n_frames(n)
    xp = np.pad(x, do.PAD + 1, mode="reflect")
    idx = do.HOP * np.arange(F)[:, None] + np.arange(do.N_FFT)[None, :] + 1 + shift
    fw = xp[idx] * w
    X = torch.fft.fft(torch.from_numpy(fw).to(torch.complex64), dim=1)[:, : do.N_BINS]
    re, im = X.real.numpy(), X.imag.numpy()
    if bf16_spectra:
        re, im = to_bf16(re), to_bf16(im)
    mag = np.sqrt(re * re + im * im).astype(np.float32)
    sb = np.float32(s) * np.asarray(bias, np.float32)
    keep = np.maximum(mag - sb[None, :], np.float32(0))
    gain = np.divide(keep, mag, out=np.zeros_like(mag), where=mag > 0).astype(np.float32)
    Y = torch.complex(torch.from_numpy(re * gain), torch.from_numpy(im * gain))
    full = torch.cat([Y, torch.conj(Y[:, 1: do.N_BINS - 1]).flip(1)], dim=1)
    yf = (torch.fft.fft(torch.conj(full), dim=1).real.numpy() * np.float32(1.0 / do.N_FFT)) * w
    acc = np.zeros(do.N_FFT + do.HOP * (F - 1), np.float32)
    env = np.zeros_like(acc)
    w2 = w.astype(np.float64) ** 2
    for f in range(F):
        sl = slice(do.HOP * f, do.HOP * f + do.N_FFT)
        acc[sl] = acc[sl] + yf[f]
        env[sl] = (w2 + env[sl].astype(np.float64)).astype(np.float32)
    return acc[do.PAD: do.PAD + n] / env[do.PAD: do.PAD + n]


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("s", STRENGTHS)
def test_oracle_equals_torch_stft_istft(n, s):
    x = signal_of(n, n)
    bias = hiss_bias()
    y = do.denoise(x, s, bias)
    assert y.shape == (n,)
    assert np.abs(y - torch_reference(x, s, bias)).max() <= 1e-12


def test_oracle_random_lengths():
    rng = np.random.default_rng(5)
    bias = hiss_bias(2)
    for n in rng.integers(513, 20000, size=12):
        x = signal_of(int(n), int(n))
        s = float(rng.choice(STRENGTHS))
        assert np.abs(do.denoise(x, s, bias) - torch_reference(x, s, bias)).max() <= 1e-12, (n, s)


@pytest.mark.parametrize("n", LENGTHS + [3001])
def test_zero_strength_reconstructs(n):
    x = signal_of(n, 7)
    assert np.abs(do.denoise(x, 0.0, hiss_bias()) - x.astype(np.float64)).max() <= 1e-12


@pytest.mark.parametrize("n", [0, 1, 2, 300, 511, 512])
def test_short_rows_are_returned_unchanged(n):
    x = signal_of(max(n, 1), 3)[:n]
    assert np.array_equal(do.denoise(x, 1.0, hiss_bias()), x.astype(np.float64))


def test_bias_equals_torch_stft_frame0():
    wav = signal_of(22528, 9)
    w = torch.hann_window(do.N_FFT, periodic=True, dtype=torch.float64)
    X = torch.stft(torch.from_numpy(wav.astype(np.float64)), do.N_FFT, do.HOP, window=w, center=True, pad_mode="reflect",
                   return_complex=True)
    b = do.bias_of(wav)
    assert b.shape == (do.N_BINS,)
    assert np.abs(b - X[:, 0].abs().numpy()).max() <= 1e-12


def test_frame_count_and_coverage():
    for n in (513, 767, 768, 1024, 80128):
        F = do.n_frames(n)
        assert do.frames(np.zeros(n)).shape == (F, do.N_FFT)
        env = do.envelope(n)
        assert env.min() > 0.2          # every output is covered by frames with real weight (least at the tail)


def test_stream_emission_formula_matches_counting():
    """after P inputs, the closed form (what the library computes) equals the count of outputs that are final whatever
    the row's final length, for every P <= 5000"""
    for P in range(0, 5001):
        assert do.emitted_closed_form(P) == do.emitted(P), P
    for P in (79872, 80128, 5_000_000 + 7):
        e = do.emitted_closed_form(P)
        assert e == 0 or do.final_after(e - 1, P)
        assert not do.final_after(e, P)
    pushes = [1, 255, 256, 1000, 0, 3000]
    assert sum(do.schedule(pushes)) == sum(pushes)
    assert do.schedule([1023, 1], end_last=False) == [0, 256]      # the 1024th sample completes frame 2
    assert do.schedule([1023, 1]) == [0, 1024]


def test_stream_lookahead_is_the_maximum_over_outputs():
    t = np.arange(100_000, dtype=np.int64)
    assert do.lookahead() == int((do.last_input(t) - t).max()) == do.LOOKAHEAD == 1023
    # the output that waits longest is the first of each hop: it reads frame t / 256 + 2 up to its end
    assert do.last_input(256) - 256 == 1023 and do.last_input(511) - 511 == 768


def test_bound_has_headroom_over_the_emulation():
    """TOL is at least 4x the worst fp32 emulation of the kernels and at least 10x below what spectra rounded to bf16,
    or frames shifted by one sample, would give"""
    worst, worst_bf, worst_shift = 0.0, np.inf, np.inf
    bias = hiss_bias()
    for n in (513, 1025, 3001, 80128):
        x = signal_of(n, n + 1)
        for s in STRENGTHS:
            y64 = do.denoise(x, s, bias)
            scale = do.error_scale(x, s, bias)
            e32 = np.abs(emulate(x, s, bias) - y64) / scale
            worst = max(worst, float(e32.max()))
            if n == 80128:
                worst_bf = min(worst_bf, float((np.abs(emulate(x, s, bias, bf16_spectra=True) - y64) / scale).max()))
                worst_shift = min(worst_shift, float((np.abs(emulate(x, s, bias, shift=1) - y64) / scale).max()))
    print(f"fp32 emulation {worst:.2e}, bf16 spectra {worst_bf:.2e}, frames shifted by one {worst_shift:.2e} (TOL {TOL:.0e})")
    assert 4 * worst <= TOL, worst
    assert worst_bf >= 10 * TOL, worst_bf
    assert worst_shift >= 10 * TOL, worst_shift
