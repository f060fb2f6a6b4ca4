"""CPU: the de-esser's definition (oracle/deesser_oracle.py), its detector as block maps, the tolerance the GPU tests hold
the device to, the spec parser, the AudioChain stage order and the CLI's argument errors.

TOL bounds error_units(y), the per-sample error of y = x - (1 - g) h against float64 in units of

    u[t] = 2^-24 (3 |y64| + |h64| (3 + (ln 10 / 20) Lam (1 + sqrt(1 / (1 - a_R)) + sqrt(1 / (1 - a_A)))))
           + dh (1 + |h64[t]| / floor),   dh = 2^-24 max |x| ||hp||_1,  floor = 10^((T - W/2) / 20).

The first line is the compressor's unit (tests/test_compressor_cpu.py) with the gain acting on h instead of on the
output: an error of e dB in y_L moves y by (ln 10 / 20) e g |h|; the 3 |y64| covers the rounding of fmaf(g - 1, h, x)
and the 3 |h64| exp10f and g - 1.  dh is the equalizer's unit (tests/test_eq_cpu.py) for the one high-pass section: it
reaches y directly through (1 - g) h <= h, and the level through 20 log10 |h|, which the detector only reads where
x_L > 0, i.e. where |h| keeps the knee's lower edge `floor`; there an error dh in h moves L by (20 / ln 10) dh / floor dB
and y by at most |h| dh / floor.  TOL is pinned against an fp32 numpy emulation of the kernels (eq_oracle.emulate for h,
the compressor test's block scans for y_L, then the apply), and every wrong variant in `VARIANTS` exceeds it."""
import numpy as np
import pytest

from oracle import compressor_oracle as co
from oracle import deesser_oracle as do
from oracle import eq_oracle as eo
from test_compressor_cpu import consts, fma, level_steps, reduction32, speech_like

TOL = 4.0            # error_units (see test_tolerance_has_headroom_over_the_emulation)
F = np.float32

PARAMS = {
    "voice": {},
    "hard": dict(knee=0.0, freq=4000.0),
    "deep": dict(ratio=20.0, threshold=-40.0, range=24.0),
    "fast": dict(attack=0.5, release=5.0, knee=12.0, freq=6000.0),
    "slow": dict(attack=20.0, release=500.0, threshold=-45.0, range=6.0),
}


# ---- signals ---------------------------------------------------------------------------------------------------------

def hiss(n, rate, seed=0):
    """noise band-limited to 5.5-7.5 kHz (the sibilant band the model's 8 kHz audio carries), unit RMS"""
    from scipy import signal
    sos = signal.butter(6, [5500, min(7500, 0.49 * rate)], "bandpass", fs=rate, output="sos")
    v = signal.sosfilt(sos, np.random.default_rng(seed).standard_normal(n + 2000))[2000:]
    return v / max(np.sqrt(np.mean(v ** 2)), 1e-30)


def sibilant_speech(n, rate, seed=0, burst_db=-12.0):
    """vowel-like harmonics of 150 Hz up to 3 kHz at -12 dBFS peak, with 60-120 ms bursts of `hiss` at burst_db RMS every
    300 ms from 20 ms on; returns (x, mask of the burst samples)"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    v = sum(np.sin(2 * np.pi * 150 * k * t + rng.uniform(0, 2 * np.pi)) / k for k in range(1, 21))
    v = 10 ** (-12 / 20) * v / np.abs(v).max() * np.minimum(1.0, t / 0.01)     # a 10 ms fade-in: no onset click
    mask = np.zeros(n, bool)
    s = int(0.02 * rate)
    while s < n:
        mask[s:s + int(rng.uniform(0.06, 0.12) * rate)] = True
        s += int(0.3 * rate)
    k = int(0.005 * rate) + 1
    env = np.convolve(mask.astype(float), np.hanning(k))[k // 2:k // 2 + n]
    env /= max(env.max(), 1e-30)
    x = v + 10 ** (burst_db / 20) * env * hiss(n, rate, seed + 1)
    return x.clip(-1, 1).astype(F), mask


def hf_tone(n, rate):
    """a steady 6 kHz sine at -6 dBFS peak: the detector settles"""
    return 0.5 * np.sin(2 * np.pi * 6000 / rate * np.arange(n))


def cases(rate, n):
    return [sibilant_speech(n, rate, rate)[0], level_steps(n, rate, rate), sibilant_speech(n, rate, 7, -3.0)[0],
            speech_like(n / rate + 0.01, rate, 3)[:n], hf_tone(n, rate), np.zeros(n)]


# ---- fp32 emulation of deesser.cu ------------------------------------------------------------------------------------

def detector32(h, c):
    """y_L of the compressor's kernels (compressor.cu's block folds, chains and refolds) on the level source h"""
    n = h.size
    nb = -(-n // co.Q)
    hb = np.zeros(nb * co.Q, F)
    hb[:n] = h
    xl = reduction32(hb.reshape(nb, co.Q), c)
    ninf = np.full(nb, -np.inf, F)

    def rel_fold(M, v):
        e = (c["bR"] * v).astype(F)
        return np.maximum(v, fma(c["aR"], M[0], e)), (c["aR"] * M[1]).astype(F), fma(c["aR"], M[2], e)

    def att_fold(M, v):
        return ninf, (c["aA"] * M[1]).astype(F), fma(c["aA"], M[2], (c["bA"] * v).astype(F))

    def apply(M, d):
        return np.maximum(M[0], fma(M[1], d, M[2]))

    def chain(M):
        d = np.zeros(nb, F)
        for i in range(1, nb):
            d[i] = apply((M[0][i - 1:i], M[1][i - 1:i], M[2][i - 1:i]), d[i - 1:i])[0]
        return d

    ident = (ninf, np.ones(nb, F), np.zeros(nb, F))
    R = ident
    for j in range(co.Q):
        R = rel_fold(R, xl[:, j])
    y1_in = chain(R)
    R, A = ident, ident
    for j in range(co.Q):
        R = rel_fold(R, xl[:, j])
        A = att_fold(A, apply(R, y1_in))
    yl_in = chain(A)
    R, A = ident, ident
    yl = np.empty((nb, co.Q), F)
    for j in range(co.Q):
        R = rel_fold(R, xl[:, j])
        A = att_fold(A, apply(R, y1_in))
        yl[:, j] = apply(A, yl_in)
    return yl.reshape(-1)[:n]


def emulate(x, rate, **kw):
    """y of deesser.cu's one-shot arithmetic in fp32 numpy"""
    p = do.params(rate, **kw)
    x = np.asarray(x, F)
    if x.size == 0:
        return x.copy()
    h = eo.emulate(do.highpass(p["freq"], rate), x)
    ylc = np.minimum(detector32(h, consts(p)), F(p["range"]))
    g = np.where(ylc > 0, np.power(F(10), (-ylc / F(20)).astype(F)), F(1)).astype(F)
    return np.where(ylc > 0, fma((g - F(1)).astype(F), h, x), x).astype(F)


def error_units(y, ref, x, P):
    """max |y - ref| / u[t] over the row (see the module docstring); P the oracle's parts"""
    y = np.asarray(y, np.float64)
    if y.size == 0:
        return 0.0
    L, h = P["L"], np.abs(P["h"])
    floor = 10.0 ** ((P["threshold"] - P["knee"] / 2) / 20)
    above = np.isfinite(L) & (L >= P["threshold"] - P["knee"] / 2)
    lam = float(np.abs(L[above]).max()) if above.any() else 0.0
    k = np.log(10) / 20 * lam * (1 + np.sqrt(1 / (1 - P["aR"])) + np.sqrt(1 / (1 - P["aA"])))
    dh = 2.0 ** -24 * float(np.abs(np.asarray(x, np.float64)).max()) * eo.impulse_l1(do.highpass(P["freq"], P["rate"]))
    u = 2.0 ** -24 * (3 * np.abs(ref) + h * (3 + k)) + dh * (1 + h / floor)
    err = np.abs(y - ref)
    if np.any((u == 0) & (err > 0)):
        return np.inf
    return float(np.max(np.where(u > 0, err / np.where(u > 0, u, 1), 0.0)))


def parts(x, rate, **kw):
    ref, red, P = do.deess(x, rate, parts=True, **kw)
    return ref, red, dict(P, rate=rate)


# ---- wrong variants of the definition (float64) ----------------------------------------------------------------------

def unwarped_highpass(freq, rate):
    """the Butterworth section through the bilinear transform without prewarping (K = pi f0 / r instead of tan)"""
    K = np.pi * freq / rate
    a0 = 1 + np.sqrt(2) * K + K * K
    return np.array([[1 / a0, -2 / a0, 1 / a0, 1.0, 2 * (K * K - 1) / a0, (1 - np.sqrt(2) * K + K * K) / a0]])


def variant(x, rate, kind, **kw):
    """y of the oracle with one deliberate mistake"""
    p = do.params(rate, **kw)
    x64 = np.asarray(x, F).astype(np.float64)
    sos = unwarped_highpass(p["freq"], rate) if kind == "nowarp" else do.highpass(p["freq"], rate)
    h = eo.sosfilt(sos, x64)
    with np.errstate(divide="ignore"):
        L = 20 * np.log10(np.abs(x64 if kind == "fullband" else h))
    xl = co.reduction(L, p["threshold"], p["ratio"], p["knee"])
    aR, bR, aA, bA = p["aR"], p["bR"], p["aA"], p["bA"]
    if kind == "swap":
        aR, bR, aA, bA = aA, bA, aR, bR
    yl = co.attack(co.release(xl, aR, bR), aA, bA)
    if kind != "norange":
        yl = np.minimum(yl, p["range"])
    g = 10.0 ** (-yl / 20)
    return g * x64 if kind == "wideband" else x64 - (1 - g) * h


VARIANTS = ("fullband", "wideband", "norange", "swap", "nowarp")


# ---- the definition --------------------------------------------------------------------------------------------------

def test_highpass_is_the_equalizers_section():
    from viettts_b200.engine import eq_sections
    for rate in (16000, 44100, 48000):
        for freq in (1000.0, 5000.0, 0.45 * rate):
            sos = do.highpass(freq, rate)
            assert sos.shape == (1, 6)
            assert np.allclose(sos, eq_sections(f"hp:{co.f32(freq)}:2", rate), rtol=0, atol=1e-12)
            w, H = __import__("scipy").signal.sosfreqz(sos, [freq], fs=rate)
            assert abs(abs(H[0]) - np.sqrt(0.5)) < 1e-9          # -3 dB at the crossover


@pytest.mark.parametrize("t0", [0, 1, 100, 255, 256, 1000])
def test_block_maps_equal_the_recursion(t0):
    rate = 16000
    x, _ = sibilant_speech(5 * co.Q + 77, rate, 5, -6.0)
    _, _, P = do.deess(x, rate, parts=True, range=6.0)
    assert np.allclose(do.yl_by_maps(P["xl"], P, t0), P["ylc"], rtol=0, atol=1e-12)
    assert P["yl"].max() > 6.0 and P["ylc"].max() == 6.0


def test_low_band_passes_and_pass_through_is_bit_exact():
    rate = 16000
    x, _ = sibilant_speech(16000, rate, 2, -6.0)
    y, red, P = do.deess(x, rate, parts=True)
    assert red < -3
    assert np.allclose(y - P["g"] * P["h"], x.astype(np.float64) - P["h"], rtol=0, atol=1e-12)    # x - h untouched
    lows = (0.05 * np.sin(2 * np.pi * 300 / rate * np.arange(8000))).astype(F)     # no high band above the knee
    for xx, kw in ((lows, {}), (x, dict(ratio=1.0)), (x, dict(range=0.0))):
        y, red = do.deess(xx, rate, **kw)
        assert red == 0.0 and np.array_equal(y, xx.astype(np.float64)), kw
        assert np.array_equal(emulate(xx, rate, **kw), xx), kw


def clear_of_bursts(mask, rate, after=0.15):
    """the samples 10 ms or more before the first burst and those at least `after` seconds past a burst's end (a 5 ms
    release has taken fp32's g back to 1 by then)"""
    c = np.concatenate([[0], np.cumsum(mask)])
    t = np.arange(mask.size)
    lead = int(0.01 * rate)                       # the bursts' 5 ms fade starts before the mask
    return c[np.minimum(t + lead + 1, mask.size)] == c[np.maximum(t - int(after * rate), 0)]


def test_bursts_are_turned_down_and_the_rest_is_not():
    rate = 48000
    x, mask = sibilant_speech(rate, rate, 4, -6.0)
    kw = dict(release=5.0)
    y, red, P = do.deess(x, rate, parts=True, **kw)
    assert -12.0 <= red < -6.0
    off = clear_of_bursts(mask, rate)
    assert off.sum() > 0.1 * rate and np.all(P["ylc"][off] < 1e-6)
    assert np.array_equal(emulate(x, rate, **kw)[off], x[off])
    high = y - (x.astype(np.float64) - P["h"])               # the split's high band of y: g h
    assert np.sum(high[mask] ** 2) < 10 ** (-6 / 10) * np.sum(P["h"][mask] ** 2)


# ---- the tolerance ---------------------------------------------------------------------------------------------------

def worst_emulation(rate, n, names=tuple(PARAMS)):
    worst = 0.0
    for name in names:
        for x in cases(rate, n):
            x = np.asarray(x, F)
            ref, _, P = parts(x, rate, **PARAMS[name])
            worst = max(worst, error_units(emulate(x, rate, **PARAMS[name]), ref, x, P))
    return worst


def test_tolerance_has_headroom_over_the_emulation():
    worst = max(worst_emulation(rate, n) for rate, n in ((16000, 12000), (44100, 20000), (48000, 30000)))
    print(f"fp32 emulation {worst:.3f} units (TOL {TOL})")
    assert 4 * worst <= TOL, worst


def test_every_wrong_variant_exceeds_the_tolerance():
    """each variant moves at least one case of the GPU tests past TOL"""
    got = {}
    for kind in VARIANTS:
        for rate, n in ((16000, 12000), (48000, 48000)):
            for name, kw in PARAMS.items():
                for x in cases(rate, n)[:5]:
                    x = np.asarray(x, F)
                    ref, _, P = parts(x, rate, **kw)
                    got[kind] = max(got.get(kind, 0.0), error_units(variant(x, rate, kind, **kw), ref, x, P))
    print({k: f"{v:.1f}" for k, v in got.items()})
    for kind in VARIANTS:
        assert got[kind] > TOL, (kind, got[kind])


# ---- spec parsing, the chain order and the CLI -----------------------------------------------------------------------

def test_spec_parsing():
    from viettts_b200.engine import DEESSER_PRESETS, deesser_params
    voice = DEESSER_PRESETS["voice"]
    assert voice == do.VOICE
    assert deesser_params("voice", 16000) == voice
    assert list(deesser_params("voice", 48000)) == ["freq", "threshold", "ratio", "knee", "attack", "release", "range"]
    p = deesser_params("freq=6500, range=6 ,ratio=8", 48000)
    assert p == dict(voice, freq=6500.0, range=6.0, ratio=8.0) and list(p) == list(voice)
    assert deesser_params({"freq": 3000, "threshold": -40}, 8000) == dict(voice, freq=3000.0, threshold=-40.0)
    assert deesser_params("freq=7200", 16000)["freq"] == 7200.0
    for k, v in deesser_params("freq=1000,threshold=-60,ratio=20,knee=24,attack=200,release=5,range=24", 192000).items():
        assert v == float(F(v))


@pytest.mark.parametrize("spec,rate,key", [("voice", 8000, "freq"), ("freq=7201", 16000, "freq"), ("freq=999", 48000, "freq"),
                                          ("range=25", 16000, "range"), ("range=-1", 16000, "range"),
                                          ("ratio=0.5", 16000, "ratio"), ("threshold=1", 16000, "threshold"),
                                          ("knee=30", 16000, "knee"), ("attack=0.1", 16000, "attack"),
                                          ("release=6000", 16000, "release"), ("range=nan", 16000, "range"),
                                          ("makeup=3", 16000, "makeup"), ("freq=abc", 16000, "freq"), ("soft", 16000, "soft"),
                                          ({"freq": float("inf")}, 16000, "freq"), ("voice", 7999, "rate")])
def test_spec_rejections_name_the_key(spec, rate, key):
    from viettts_b200.engine import deesser_params
    with pytest.raises(ValueError, match=key):
        deesser_params(spec, rate)


def test_audio_chain_stage_order():
    from viettts_b200.engine import AudioChain, OptionError
    ch = AudioChain(output_rate=48000, eq="hs:6000:3", compress="voice", deess="voice", limit=-1.0, meter=True)
    assert [s[0] for s in ch._stages()] == ["rs", "eq", "cp", "ds", "lm", "mt"]
    ch = AudioChain(deess="range=6", loudness=-16.0, limit=-1.0)
    assert [s[0] for s in ch._stages()] == ["ds", "lm"]
    assert ch.deess["range"] == 6.0
    assert [s[0] for s in AudioChain(deess="voice", denoise=0.5, compress="voice")._stages()] == ["dn", "cp", "ds"]
    assert AudioChain().deess is None and [s[0] for s in AudioChain(compress="voice")._stages()] == ["cp"]
    with pytest.raises(OptionError) as e:
        AudioChain(deess="voice", output_rate=8000)
    assert e.value.option == "deess" and "freq" in str(e.value)


@pytest.mark.parametrize("argv", [["--deess", "range=30"], ["--deess", "harsh"], ["--deess", "freq=200"],
                                  ["--deess", "voice", "--output-rate", "8000"], ["--deess", "knee=x"]])
def test_cli_rejects_bad_deess(argv, capsys):
    from viettts_b200 import synthesizer
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
    assert "--deess" in capsys.readouterr().err
