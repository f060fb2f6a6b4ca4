"""CPU: the resampler's definition, its filter design, its stream schedule and the tolerance the GPU tests hold it to.

The oracle (oracle/resample_oracle.py) is pinned against scipy.signal.resample_poly; the library's double-precision
design (vtts_resample_filter) against scipy.signal.firwin; the stream lookahead and emission formula against the
oracle's counting; and TOL -- the bound |y - y64| <= TOL * sum|h x| per output -- against a numpy emulation of the
kernel's fp32 sum order."""
import ctypes as C

import numpy as np
import pytest
from scipy import signal

from oracle import resample_oracle as ro

SR = 16000
RATES = [(SR, r) for r in (8000, 11025, 22050, 24000, 32000, 44100, 48000)] + [(48000, SR)]
LENGTHS = [1, 2, 9, 255, 256, 257, 79872]
TOL = 2e-6    # per output, relative to sum |h x| (see test_bound_has_headroom_over_the_emulation)


def signal_of(n, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    return (0.5 * np.sin(2 * np.pi * 440 * t) + 0.3 * rng.standard_normal(n)).astype(np.float32)


def to_bf16(a):
    u = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return u.view(np.float32)


def emulate(x, in_rate, out_rate, h32):
    """the kernel's arithmetic in numpy: per output the T-term sum in ascending input index, the first term a product,
    every later one an FMA (exact product, one rounding to fp32), inputs outside [0, n) and taps past 2 * half zero"""
    x = np.asarray(x, np.float32)
    up, down, half = ro.ratio(in_rate, out_rate)
    n = x.size
    T = -(-(2 * half + 1) // up)
    m = np.arange(ro.out_len(n, in_rate, out_rate), dtype=np.int64)
    j = m * down + half
    top = j // up
    h = np.asarray(h32, np.float32)
    acc = None
    for t in range(T):
        i = top - (T - 1) + t
        k = j - i * up
        xv = np.where((i >= 0) & (i < n), x[np.clip(i, 0, n - 1)], np.float32(0)).astype(np.float64)
        hv = np.where(k <= 2 * half, h[np.clip(k, 0, 2 * half)], np.float32(0)).astype(np.float64)
        acc = (xv * hv).astype(np.float32) if acc is None else (xv * hv + acc.astype(np.float64)).astype(np.float32)
    return acc


def library_filter(in_rate, out_rate):
    from viettts_b200 import _lib
    lib = _lib.load()
    n = lib.vtts_resample_filter(in_rate, out_rate, None, 0)
    assert n > 0
    h = np.zeros(n)
    assert lib.vtts_resample_filter(in_rate, out_rate, h.ctypes.data_as(C.c_void_p), n) == n
    return h


@pytest.mark.parametrize("rates", RATES, ids=lambda r: f"{r[0]}-{r[1]}")
@pytest.mark.parametrize("n", LENGTHS)
def test_oracle_equals_resample_poly(rates, n):
    x = signal_of(n, n)
    up, down, _ = ro.ratio(*rates)
    ref = signal.resample_poly(x.astype(np.float64), up, down)
    y = ro.resample(x, *rates)
    assert y.shape == ref.shape == (ro.out_len(n, *rates),)
    assert np.abs(y - ref).max() <= 1e-12


def test_oracle_copy_when_rates_match():
    x = signal_of(300)
    assert np.array_equal(ro.resample(x, SR, SR), x.astype(np.float64))


@pytest.mark.parametrize("rates", RATES, ids=lambda r: f"{r[0]}-{r[1]}")
def test_library_filter_equals_firwin(rates):
    up, down, half = ro.ratio(*rates)
    h = library_filter(*rates)
    ref = signal.firwin(2 * half + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up
    assert h.shape == ref.shape
    assert np.abs(h - ref).max() <= 1e-12
    assert np.abs(h - ro.design(*rates)).max() <= 1e-12


def test_library_filter_arguments():
    from viettts_b200 import _lib
    lib = _lib.load()
    assert list(library_filter(SR, SR)) == [1.0]
    assert lib.vtts_resample_filter(SR, 48000, None, 0) == 61
    assert lib.vtts_resample_filter(SR, 11025, None, 0) == 12801
    small = np.full(4, 7.0)
    assert lib.vtts_resample_filter(SR, 48000, small.ctypes.data_as(C.c_void_p), 4) == 61
    assert np.all(small == 7.0)                                   # too small: nothing written
    for a, b in ((0, SR), (SR, 0), (-SR, 48000), (SR, 1031), (1031, 1033)):
        assert lib.vtts_resample_filter(a, b, None, 0) == -1, (a, b)
        assert lib.vtts_resample_stream_lookahead(a, b) == -1, (a, b)


@pytest.mark.parametrize("rates", RATES + [(SR, SR)], ids=lambda r: f"{r[0]}-{r[1]}")
def test_stream_lookahead(rates):
    from viettts_b200 import _lib
    lib = _lib.load()
    up, _, half = ro.ratio(*rates)
    assert lib.vtts_resample_stream_lookahead(*rates) == ro.lookahead(*rates) == half // up
    expect = {8000: 20, 11025: 14, 22050: 10, 24000: 10, 44100: 10, 48000: 10}
    if rates[0] == SR and rates[1] in expect:
        assert ro.lookahead(*rates) == expect[rates[1]]


@pytest.mark.parametrize("rates", RATES + [(SR, SR)], ids=lambda r: f"{r[0]}-{r[1]}")
def test_emission_formula_matches_counting(rates):
    """after P inputs, the closed form (what the library computes) equals the count of outputs whose last input has
    arrived: every output appears with exactly the push that brings its last input, not one push later"""
    up, down, half = ro.ratio(*rates)
    Ps = list(range(0, 3000)) + [79872, 5_000_000 + 7]
    for P in Ps:
        e = ro.emitted_closed_form(P, *rates)
        if P < 3000:
            assert e == ro.emitted(P, *rates), P
        # tight: output e - 1 has its last input before P, output e has not (or does not exist yet)
        if e > 0:
            assert ro.last_input(e - 1, *rates) <= P - 1
        assert e == ro.out_len(P, *rates) or ro.last_input(e, *rates) >= P
    # pushes emit their outputs in order, and END the rest
    pushes = [1, 3, 10, 256, 1, 0, 700]
    sched = ro.schedule(pushes, *rates)
    assert sum(sched) == ro.out_len(sum(pushes), *rates)


def test_bound_has_headroom_over_the_emulation():
    """TOL is at least 4x the worst fp32 emulation of the kernel (fp32 taps, its sum order) and at least 10x below what
    taps rounded to bf16 would give"""
    worst, worst_bf = 0.0, np.inf
    for rates in RATES:
        x = signal_of(20000, 3)
        y64 = ro.resample(x, *rates)
        scale = np.maximum(ro.abs_sum(x, *rates), 1e-30)
        h = ro.design(*rates)
        e32 = np.abs(emulate(x, *rates, h.astype(np.float32)) - y64) / scale
        ebf = np.abs(emulate(x, *rates, to_bf16(h.astype(np.float32))) - y64) / scale
        print(f"{rates}: fp32 emulation {e32.max():.2e}, bf16 taps {ebf.max():.2e} (TOL {TOL:.0e})")
        worst = max(worst, float(e32.max()))
        worst_bf = min(worst_bf, float(ebf.max()))
    assert 4 * worst <= TOL, worst
    assert worst_bf >= 10 * TOL, worst_bf


def test_python_ratio_helpers():
    from viettts_b200.engine import resample_length, resample_ratio
    assert resample_ratio(SR, 44100) == (441, 160)
    assert resample_ratio(SR, 11025) == (441, 640)
    assert resample_length(79872, SR, 44100) == ro.out_len(79872, SR, 44100) == 220148   # ceil(220147.2)
    with pytest.raises(ValueError):
        resample_ratio(SR, 0)
