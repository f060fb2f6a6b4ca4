"""CPU: the limiter's definition (oracle/limiter_oracle.py), its release scan as maps, its stream schedule, the tolerance
the GPU tests hold the device to, and the CLI's argument errors.

Y_TOL -- the bound on error_units(y), the error of y against float64 in units of max |v| 2^-24 (1 + 1 / (1 - beta)) -- is
pinned against an fp32 numpy emulation of limiter.cu's arithmetic: the fp32 polyphase oversampler, the fp32 tau, the
integer-quantized box and the block scan of release maps.  The release is a leaky integrator whose memory is
1 / (1 - beta) samples, so its fp32 rounding errors add up over that many samples; the unit scales with it."""
import numpy as np
import pytest
from scipy import signal

from oracle import limiter_oracle as lm
from oracle import loudness_oracle as lo

Y_TOL = 1.0           # error_units (see test_tolerance_has_headroom_over_the_emulation)
TP_MARGIN = 0.25      # dB over the ceiling for the output's true peak; the worst of adversarial_cases is 0.15 dB


def fs4_sine(n, amp=1.0):
    return amp * np.sin(np.pi / 2 * np.arange(n) + np.pi / 4)


def clicks(n):
    x = np.zeros(n)
    x[n // 3] = 1.0
    x[n // 2] = -1.0
    x[n // 2 + 3] = 0.7
    return x


def noise(n, seed=0, amp=0.5):
    return amp * np.random.default_rng(seed).standard_normal(n)


def burst(n, rate):
    x = np.zeros(n)
    d = rate // 50
    x[n // 4:n // 4 + d] = np.sin(2 * np.pi * 3000 / rate * np.arange(d))
    return x


def speech_like(seconds, rate, seed=0):
    """AR(1) noise under a random syllable envelope: a peak-to-loudness ratio near that of speech"""
    rng = np.random.default_rng(seed)
    n = int(seconds * rate)
    e = signal.lfilter([1.0], [1.0, -0.9], rng.standard_normal(n))
    env = np.zeros(n)
    t = 0
    while t < n:
        d = int(rng.uniform(0.08, 0.3) * rate)
        env[t:t + d] = rng.uniform(0.05, 1.0) * np.hanning(d)[: n - t]
        t += d + int(rng.uniform(0.02, 0.2) * rate)
    x = e * env
    return (0.9 * x / np.abs(x).max()).astype(np.float32)


def adversarial_cases(rate):
    n = rate // 4
    return [fs4_sine(n), clicks(n), noise(n, rate), burst(n, rate)]


# ---- fp32 emulation of limiter.cu ----------------------------------------------------------------------------------

def _taps():
    """the resampler's fp32 polyphase filter of 4 / 1: [phase][tap], tap t multiplies input it - 20 + t"""
    h = signal.firwin(81, 0.25, window=("kaiser", 5.0))
    h = h / h.sum() * 4
    T = 21
    pp = np.zeros((4, T))
    for p in range(4):
        for t in range(T):
            k = p + (T - 1 - t) * 4
            if k <= 80:
                pp[p, t] = h[k]
    return pp.astype(np.float32)


def _oversample32(v):
    f = np.float32
    n = v.size
    pp = _taps()
    xp = np.concatenate([np.zeros(20, f), v, np.zeros(20, f)])
    m = np.arange(4 * n)
    j = m + 40
    it, ph = j // 4, j % 4
    acc = xp[it - 20 + 20] * pp[ph, 0]
    for t in range(1, 21):
        acc = (acc + xp[it - 20 + t + 20] * pp[ph, t]).astype(f)
    return acc


def _round_up_f32(q):
    a = q.astype(np.float32)
    low = a.astype(np.float64) < q.astype(np.float64)
    a[low] = np.nextafter(a[low], np.float32(np.inf))
    return a


def emulate(x, rate, ceiling, gain_db=0.0, lookahead_ms=5.0, release_ms=100.0):
    """y of limiter.cu's arithmetic in fp32 numpy (no FMA: the error is of the same size)"""
    f = np.float32
    W, beta = lm.params(rate, lookahead_ms, release_ms)
    b32, omb = f(beta), f(1.0 - beta)
    c = f(10.0 ** (float(f(ceiling)) / 20.0))
    v = (lm.gain_factor(gain_db) * np.asarray(x, f)).astype(f)
    n = v.size
    g = np.abs(_oversample32(v)).reshape(n, 4).max(axis=1)
    gp = np.concatenate([np.zeros(lm.D, f), g, np.zeros(lm.D, f)])
    p = np.maximum(np.abs(v), np.lib.stride_tricks.sliding_window_view(gp, 2 * lm.D + 1).max(axis=1))
    with np.errstate(divide="ignore"):
        tau = np.where(p > 0, np.minimum(f(1), c / np.where(p > 0, p, f(1))), f(1)).astype(f)
    h = np.lib.stride_tricks.sliding_window_view(np.concatenate([tau, np.ones(W - 1, f)]), W).min(axis=1)
    q = (1 << 32) - np.floor(h.astype(np.float64) * 2.0 ** 32).astype(np.int64)
    cs = np.concatenate([[0], np.cumsum(np.concatenate([np.zeros(W - 1, np.int64), q]))])
    box = cs[W:] - cs[:-W]
    a = (_round_up_f32(-(-box // W)) * f(2.0 ** -32)).astype(f)
    d = np.empty(n, f)
    d_in = f(0)
    for b0 in range(0, n, lm.Q):
        cM, mM, kM = f(-np.inf), f(1), f(0)
        for t in range(b0, min(n, b0 + lm.Q)):
            e = f(omb * a[t])
            cM, mM, kM = max(a[t], f(f(b32 * cM) + e)), f(b32 * mM), f(f(b32 * kM) + e)
            d[t] = max(cM, f(f(mM * d_in) + kM))
        d_in = max(cM, f(f(mM * d_in) + kM))
    return (v * np.minimum(tau, (f(1) - d).astype(f))).astype(f)


def error_units(y, ref, P):
    """max |y - ref| in units of max |v| 2^-24 (1 + 1 / (1 - beta)), P the oracle's parts"""
    vmax = float(np.abs(P["v"]).max()) if P else 0.0
    if vmax == 0.0:
        return 0.0 if np.array_equal(np.asarray(y, np.float64), ref) else np.inf
    return float(np.abs(np.asarray(y, np.float64) - ref).max()) / (vmax * 2.0 ** -24 * (1.0 + 1.0 / (1.0 - P["beta"])))


# ---- the definition --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rate", [8000, 16000, 48000])
@pytest.mark.parametrize("A,R,G", [(1, 10, 0), (5, 100, 20), (20, 50, 40)])
def test_sample_and_true_peak_bounds(rate, A, R, G):
    for x in adversarial_cases(rate):
        y, red, P = lm.limit(x.astype(np.float32), rate, -1.0, G, A, R, parts=True)
        assert np.abs(y).max() <= P["c"] * (1 + 2 ** -23)
        assert lo.true_peak(y) <= -1.0 + TP_MARGIN
        assert red <= 0.0
        w = P["W"] - 1                                       # the attack window lies inside the row
        assert np.all(1.0 - P["a"][w:] <= P["tau"][w:] + 1e-12)


def test_quiet_rows_pass_through_bit_exact():
    x = (0.3 * np.sin(2 * np.pi * 440 / 16000 * np.arange(8000))).astype(np.float32)
    y, red = lm.limit(x, 16000, -1.0, 3.0)
    assert red == 0.0
    assert np.array_equal(y, float(lm.gain_factor(3.0)) * x.astype(np.float64))


@pytest.mark.parametrize("A", [1, 5, 20])
def test_attack_starts_at_most_w_plus_d_before_the_peak(A):
    rate = 16000
    x = np.zeros(4000, np.float32)
    x[2000] = 1.0
    y, _, P = lm.limit(x, rate, -6.0, 0.0, A, 100.0, parts=True)
    first = int(np.flatnonzero(P["g"] < 1.0)[0])
    assert 2000 - first <= P["W"] + lm.D
    assert P["g"][2000] <= P["tau"][2000]


def test_release_recovers_at_rate_beta():
    rate, R = 16000, 50.0
    x = np.zeros(6000, np.float32)
    x[1000:1010] = 1.0
    _, _, P = lm.limit(x, rate, -6.0, 0.0, 2.0, R, parts=True)
    d, a, beta = P["d"], P["a"], P["beta"]
    tail = np.flatnonzero(a == 0)
    tail = tail[tail > 1100][:500]
    assert np.allclose(d[tail], beta * d[tail - 1], rtol=1e-12, atol=0)
    assert d[tail[0] - 1] > 0.4


def test_folded_maps_equal_the_recurrence():
    rate = 16000
    x = noise(3 * lm.Q + 77, 3, 1.0).astype(np.float32)
    _, _, P = lm.limit(x, rate, -3.0, 0.0, 3.0, 20.0, parts=True)
    d = lm.release_by_maps(P["a"], P["beta"])
    assert np.allclose(d, P["d"], rtol=1e-12, atol=1e-15)
    # composing any split of the maps gives the map of the whole
    M = lm.IDENTITY
    for t, at in enumerate(P["a"][:300]):
        M = lm.fold(M, float(at), P["beta"], (1 - P["beta"]) * float(at))
    assert abs(lm.apply_map(M, 0.0) - P["d"][299]) < 1e-12


@pytest.mark.parametrize("W", [1, 2, 16, 80, 960])
def test_stream_lookahead_matches_counting(W):
    L = lm.stream_lookahead(W)
    assert L == W + lm.D + 9
    for P in list(range(0, 3 * L + 5)) + [5000]:
        assert lm.released(P, W) == max(0, P - L)
        assert lm.released(P, W, end=True) == P


def test_normalize_limited_reaches_a_target_the_capped_gain_misses():
    rate = 16000
    x = speech_like(6.0, rate, 1)
    L, _, _, tp = lo.measure(x, rate)
    assert tp - L > 16.0                                         # PLR over T - C = 15 dB
    capped = x.astype(np.float64) * 10 ** (lo.gain(x, rate, -16.0, -1.0) / 20)
    y, G = lm.normalize_limited(x, rate, -16.0, -1.0)
    Lc, Ly = lo.measure(capped, rate)[0], lo.measure(y, rate)[0]
    print(f"capped {Lc:.2f} LUFS, limited {Ly:.2f} LUFS, G {G:.2f} dB")
    assert Lc < -18.0
    assert Ly > Lc + 2.0 and abs(Ly + 16.0) < 1.5
    assert lo.true_peak(y) <= -1.0 + TP_MARGIN


def test_tolerance_has_headroom_over_the_emulation():
    worst = 0.0
    for rate, A, R, G in ((16000, 5, 100, 0), (48000, 2, 30, 20), (8000, 20, 10, 6)):
        for x in [fs4_sine(3000), clicks(3000), noise(3000, rate), speech_like(0.4, rate, 2)]:
            x = np.asarray(x, np.float32)
            ref, _, P = lm.limit(x, rate, -1.0, G, A, R, parts=True)
            worst = max(worst, error_units(emulate(x, rate, -1.0, G, A, R), ref, P))
    print(f"fp32 emulation {worst:.2f} units (Y_TOL {Y_TOL})")
    assert 4 * worst <= Y_TOL <= 16, worst


# ---- the CLI -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("argv", [["--true-peak", "-1"], ["--limiter", "--true-peak", "-30"], ["--limiter", "--true-peak", "nan"],
                                  ["--limiter", "--output-rate", "22051"], ["--loudness", "-16", "--limiter", "--true-peak", "1"]])
def test_cli_rejects_bad_limiter_arguments(argv):
    from viettts_b200 import synthesizer
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])


def test_engine_validators():
    from viettts_b200.engine import _gain_db, _limit_args
    assert _limit_args(-1, 16000, 5, 100) == (-1.0, 16000, 5.0, 100.0)
    for bad in ((1.0, 16000, 5, 100), (-1, 16001, 5, 100), (-1, 16000, 0.5, 100), (-1, 16000, 5, 3000), (float("nan"), 16000, 5, 100)):
        with pytest.raises(ValueError):
            _limit_args(*bad)
    assert _gain_db(3, 2).tolist() == [3.0, 3.0]
    for bad in (80, float("inf"), [1, 2, 3]):
        with pytest.raises(ValueError):
            _gain_db(bad, 2)
