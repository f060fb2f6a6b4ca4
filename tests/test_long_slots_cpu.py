"""CPU companion of test_gpu_long_slots.py: the offset oracles it evaluates at a slot's absolute position reduce to the
original ones at offset 0, and the counting formulas it holds every push to stay exact at 64-bit positions."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import denoise_oracle as dn
from oracle import resample_oracle as ro
from oracle import time_stretch_oracle as tso
from oracle import watermark_oracle as wo
from test_watermark_cpu import KEY, speech

BIG = [(1 << 24) + 12345, (1 << 31) - 20000, (1 << 31) + 6789, (1 << 32) + 4321]


def test_watermark_frame_offset():
    x = speech(1.5)
    base = wo.embed(x, KEY, np.float32(0.1))
    assert np.array_equal(wo.embed(x, KEY, np.float32(0.1), frame0=0), base)
    # the chips repeat every 64 groups of 4 frames: a whole number of periods leaves the mark unchanged
    assert np.array_equal(wo.embed(x, KEY, np.float32(0.1), frame0=(1 << 33) // dn.HOP), base)
    # any other offset keys the frames with other chips
    for f0 in (wo.G, (1 << 31) // dn.HOP + wo.G):
        assert np.max(np.abs(wo.embed(x, KEY, np.float32(0.1), frame0=f0) - base)) > 1e-3 * np.abs(x).max()


@pytest.mark.parametrize("tempo", [0.5, 0.75, 0.9, 1.25, 1.37, 1.6180339, 2.0])
def test_stretch_scanned_by_bisection(tempo):
    """the bisection equals the linear scan of its definition"""
    a = tso.tempo_of(tempo)

    def linear(P):
        if P <= tso.PAD:
            return 0
        q = 0
        while int(np.rint(256.0 * q * a)) + tso.PAD <= P:
            q += 1
        return q
    rng = np.random.default_rng(3)
    for P in list(range(0, 2000, 7)) + [int(v) for v in rng.integers(0, 200_000, 60)]:
        assert tso.stretch_scanned(P, tempo) == linear(P), P


@pytest.mark.parametrize("tempo", [0.75, 0.9, 1.25, 1.37])
def test_stretch_counts_at_64bit_positions(tempo):
    """256 alpha = p / q in lowest terms.  The centres rint(256 t alpha) round halves to even, so they repeat after q
    frames and p inputs when q = 1 and after 2q and 2p otherwise: that many more inputs scan that many more frames and,
    at END, make 256 times as many more outputs, at any position.  The scanned count is the largest Q with
    rint(256 (Q - 1) alpha) + 512 <= P"""
    r = Fraction(float(np.float32(tempo))) * 256
    k = 1 if r.denominator == 1 else 2
    p, q = k * r.numerator, k * r.denominator
    a = tso.tempo_of(tempo)
    t = np.arange(0, 4 * q, dtype=np.int64) + (1 << 30)
    assert np.array_equal(np.rint(256.0 * (t + q) * a) - np.rint(256.0 * t * a), np.full(t.size, float(p)))
    for P in BIG:
        Q = tso.stretch_scanned(P, tempo)
        assert int(np.rint(256.0 * (Q - 1) * a)) + tso.PAD <= P < int(np.rint(256.0 * Q * a)) + tso.PAD
        s = P % p + 2 * p
        assert Q - tso.stretch_scanned(s, tempo) == (P - s) // p * q
        assert tso.stretch_emitted(P, tempo, True) - tso.stretch_emitted(s, tempo, True) == (P - s) // p * q * 256


def test_stretch_half_period_fails_at_exact_halves():
    """why the period doubles: at tempo 0.9 (256 alpha = 7549747 / 32768) a shift by one odd p moves every exact half
    t = 16384 (mod 32768) to the other even neighbour"""
    r = Fraction(float(np.float32(0.9))) * 256
    p, q = r.numerator, r.denominator
    a = tso.tempo_of(0.9)
    t = np.array([q // 2, q // 2 + 5 * q], np.int64)
    assert np.all(np.abs(np.rint(256.0 * (t + q) * a) - np.rint(256.0 * t * a) - p) == 1)


@pytest.mark.parametrize("rates", [(22050, 48000), (22050, 44100), (22050, 8000), (48000, 22050)])
def test_resample_counts_at_64bit_positions(rates):
    """the stream's count min(ceil(P up / down), max(0, floor((P up - 1 - half) / down) + 1)) in Python ints: down more
    inputs give up more outputs, and the count is the outputs whose last input has arrived"""
    up, down, half = ro.ratio(*rates)
    for P in BIG:
        total = -(-P * up // down)
        e = min(total, max(0, (P * up - 1 - half) // down + 1))
        assert total == ro.out_len(P, *rates)
        s = P % down + 4 * down
        e_s = min(-(-s * up // down), (s * up - 1 - half) // down + 1)
        assert e - e_s == (P - s) // down * up
        # output e - 1 needs input floor(((e - 1) down + half) / up), which has arrived; output e needs one more
        assert ((e - 1) * down + half) // up <= P - 1 < (e * down + half) // up
