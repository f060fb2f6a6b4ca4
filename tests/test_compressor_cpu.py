"""CPU: the compressor's definition (oracle/compressor_oracle.py), its two scans as block maps, the tolerance the GPU
tests hold the device to, the spec parser, the AudioChain stage order and the CLI's argument errors.

TOL bounds error_units(y), the per-sample error of y against float64 in units of

    u[t] = 2^-24 |y64[t]| (3 + (ln 10 / 20) Lam (1 + sqrt(1 / (1 - a_R)) + sqrt(1 / (1 - a_A)))),

Lam the row's largest |L[t]| above the knee's lower edge.  The 3 covers the output's own arithmetic: exp10f (within
2 ulp) and the two products of y = (x m) g.  An error of e dB in y_L moves y by ln 10 / 20 e relative;
the level carries a rounding error of about 2^-24 Lam into x_L, and each stage is a one-pole integrator whose own
roundings, about 2^-24 of the value per sample, add up over its memory of 1 / (1 - a) samples.  Round-to-nearest
errors of opposite sign cancel, so they grow with the square root of the memory; the worst case (the linear memory)
is 20-500 times looser than what the kernels do, loose enough that a 5 s release would hide a wrong stage coefficient
(`VARIANTS`: b = fp32(1 - alpha) instead of 1 - a moves a 200 ms attack's DC gain by up to 3e-4 at 48 kHz).
TOL is pinned against an fp32 numpy emulation of compressor.cu's arithmetic (block folds, chains and refolds, fmaf as
one rounding of the exact double result), and every wrong variant in `VARIANTS` exceeds it."""
import numpy as np
import pytest
from scipy import signal

from oracle import compressor_oracle as co

TOL = 3.0            # error_units (see test_tolerance_has_headroom_over_the_emulation)
F = np.float32

PARAMS = {
    "voice": {},
    "hard": dict(knee=0.0),
    "r20": dict(ratio=20.0, threshold=-30.0),
    "fast": dict(attack=0.5, release=5.0, knee=12.0),
    "slow": dict(attack=200.0, release=5000.0, threshold=-40.0),
    "smooth": dict(attack=200.0, release=5.0, threshold=-50.0, ratio=20.0),
}


# ---- signals ---------------------------------------------------------------------------------------------------------

def noise(n, seed=0, amp=0.5):
    return amp * np.random.default_rng(seed).standard_normal(n)


def level_steps(n, rate, seed=0):
    """noise whose level steps across the knee every 50 ms: -50, -30, -20, -6, -24, -10 dBFS RMS in turn"""
    rng = np.random.default_rng(seed)
    seg = max(1, rate // 20)
    levels = np.array([-50.0, -30.0, -20.0, -6.0, -24.0, -10.0])
    lv = levels[(np.arange(n) // seg) % levels.size]
    return (10 ** (lv / 20) * rng.standard_normal(n)).clip(-1, 1)


def sine_bursts(n, rate):
    """a 440 Hz sine in 100 ms bursts at -40, -18 and -3 dBFS peak, with silence between"""
    t = np.arange(n)
    seg = max(1, rate // 10)
    amp = np.array([10 ** (-40 / 20), 0.0, 10 ** (-18 / 20), 0.0, 10 ** (-3 / 20), 0.0])[(t // seg) % 6]
    return amp * np.sin(2 * np.pi * 440 / rate * t)


def tone(n, rate):
    """a steady 440 Hz sine at -3 dBFS peak: the detector settles to its DC gain"""
    return 10 ** (-3 / 20) * np.sin(2 * np.pi * 440 / rate * np.arange(n))


def speech_like(seconds, rate, seed=0):
    """AR(1) noise under a random syllable envelope, peaking at 0.9"""
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
    return (0.9 * x / max(np.abs(x).max(), 1e-30)).astype(np.float32)


def cases(rate, n):
    return [level_steps(n, rate, rate), sine_bursts(n, rate), speech_like(n / rate + 0.01, rate, 3)[:n], tone(n, rate), np.zeros(n)]


# ---- fp32 emulation of compressor.cu ---------------------------------------------------------------------------------

def fma(a, b, c):
    """fmaf: one rounding of the exact double result"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F)


def consts(p):
    s = 1.0 - 1.0 / p["ratio"]
    return dict(T=F(p["threshold"]), hw=F(0.5) * F(p["knee"]), s=F(s), q=F(s / (2.0 * p["knee"])) if p["knee"] > 0 else F(0),
                aR=F(p["aR"]), bR=F(p["bR"]), aA=F(p["aA"]), bA=F(p["bA"]), m=F(p["m"]))


def reduction32(x, c):
    with np.errstate(divide="ignore", invalid="ignore"):
        over = (F(20) * np.log10(np.abs(np.asarray(x, F)))).astype(F) - c["T"]
        u = (over + c["hw"]).astype(F)
        xl = np.where(over > c["hw"], c["s"] * over, (c["q"] * u) * u).astype(F)
        return np.where(over >= -c["hw"], xl, F(0)).astype(F)


def emulate(x, rate, **kw):
    """y of compressor.cu's one-shot arithmetic in fp32 numpy, vectorized over the blocks"""
    p = co.params(rate, **kw)
    c = consts(p)
    x = np.asarray(x, F)
    n = x.size
    if n == 0:
        return x.copy()
    nb = -(-n // co.Q)
    xb = np.zeros(nb * co.Q, F)
    xb[:n] = x
    xb = xb.reshape(nb, co.Q)
    xl = reduction32(xb, c)
    ninf = np.full(nb, -np.inf, F)

    def rel_fold(M, v):
        cM, mM, kM = M
        e = (c["bR"] * v).astype(F)
        return np.maximum(v, fma(c["aR"], cM, e)), (c["aR"] * mM).astype(F), fma(c["aR"], kM, e)

    def att_fold(M, v):
        _, mM, kM = M
        return ninf, (c["aA"] * mM).astype(F), fma(c["aA"], kM, (c["bA"] * v).astype(F))

    def apply(M, d):
        return np.maximum(M[0], fma(M[1], d, M[2]))

    def chain(M):
        d = np.zeros(nb, F)
        for i in range(1, nb):       # every block but the last is complete
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
    yl = yl.reshape(-1)[:n]
    g = np.where(yl > 0, np.power(F(10), (-yl / F(20)).astype(F)), F(1)).astype(F)
    return ((x * c["m"]).astype(F) * g).astype(F)


def error_units(y, ref, P):
    """max |y - ref| / u[t] over the row (see the module docstring); P the oracle's parts"""
    y = np.asarray(y, np.float64)
    if y.size == 0:
        return 0.0
    L = P["L"]
    above = np.isfinite(L) & (L >= P["threshold"] - P["knee"] / 2)
    lam = float(np.abs(L[above]).max()) if above.any() else 0.0
    k = np.log(10) / 20 * lam * (1 + np.sqrt(1 / (1 - P["aR"])) + np.sqrt(1 / (1 - P["aA"])))
    u = 2.0 ** -24 * np.abs(ref) * (3 + k)
    err = np.abs(y - ref)
    if np.any((u == 0) & (err > 0)):
        return np.inf
    return float(np.max(np.where(u > 0, err / np.where(u > 0, u, 1), 0.0)))


# ---- wrong variants of the definition (float64) ----------------------------------------------------------------------

def variant(x, rate, kind, **kw):
    """y of the oracle with one deliberate mistake"""
    p = co.params(rate, **kw)
    x64 = np.asarray(x, F).astype(np.float64)
    L = co.level(x64)
    if kind == "late":
        L = np.concatenate([[-np.inf], L[:-1]])
    W = 0.0 if kind == "hard" else p["knee"]
    xl = co.reduction(L, p["threshold"], p["ratio"], W)
    aR, bR, aA, bA = p["aR"], p["bR"], p["aA"], p["bA"]
    if kind == "swap":
        aR, bR, aA, bA = aA, bA, aR, bR
    if kind == "b":
        bR = co.f32(1.0 - np.exp(-1000.0 / (p["release"] * rate)))
        bA = co.f32(1.0 - np.exp(-1000.0 / (p["attack"] * rate)))
    yl = co.attack(co.release(xl, aR, bR), aA, bA)
    return x64 * p["m"] * 10.0 ** (-yl / 20.0)


VARIANTS = ("swap", "late", "hard", "b")


# ---- the definition --------------------------------------------------------------------------------------------------

def test_gain_computer_is_eq4_continuous_and_c1():
    for T, R, W in ((-24.0, 3.0, 6.0), (-40.0, 20.0, 24.0), (-10.0, 1.5, 0.5), (-60.0, 4.0, 0.0)):
        L = np.linspace(-90, 0, 9001)
        G = co.gain_computer(L, T, R, W)
        xl = co.reduction(L, T, R, W)
        assert np.allclose(xl, L - G, rtol=0, atol=1e-12)
        assert np.all(xl >= 0) and np.all(xl[2 * (L - T) < -W] == 0)
        assert np.allclose(G[2 * (L - T) > W], T + (L[2 * (L - T) > W] - T) / R, rtol=0, atol=1e-12)
        for edge in (T - W / 2, T + W / 2):           # continuous at both knee edges
            lo, hi = co.gain_computer(np.array([edge - 1e-9, edge + 1e-9]), T, R, W)
            assert abs(hi - lo) < 1e-8
            if W > 0:                                   # and C1: the slope is 1 below, 1/R above
                h = 1e-6
                d_lo = (co.gain_computer(edge, T, R, W) - co.gain_computer(edge - h, T, R, W)) / h
                d_hi = (co.gain_computer(edge + h, T, R, W) - co.gain_computer(edge, T, R, W)) / h
                assert abs(d_hi - d_lo) < 1e-4, (T, R, W, edge)
    assert co.reduction(np.array([-np.inf]), -24.0, 3.0, 6.0)[0] == 0.0
    L = np.linspace(-90, 0, 901)
    assert np.all(co.reduction(L, -30.0, 1.0, 6.0) == 0) and np.all(co.reduction(L, -30.0, 1.0, 0.0) == 0)


def test_coefficients_are_exact_complements():
    for rate in (8000, 16000, 44100, 48000, 192000):
        for tau in (0.5, 5.0, 80.0, 200.0, 5000.0):
            a, b = co.coeff(tau, rate)
            assert a >= 0.778 and b == 1.0 - a and F(b) == F(1) - F(a)


@pytest.mark.parametrize("t0", [0, 1, 100, 255, 256, 1000])
def test_block_maps_equal_the_recursion(t0):
    rate = 16000
    x = speech_like(0.2, rate, 5)[: 5 * co.Q + 77]
    _, _, P = co.compress(x, rate, parts=True, attack=2.0, release=30.0, threshold=-30.0)
    y1 = co.release_by_maps(P["xl"], P["aR"], P["bR"], t0)
    assert np.allclose(y1, P["y1"], rtol=0, atol=1e-12)
    yl = co.attack_by_maps(P["y1"], P["aA"], P["bA"], t0)
    assert np.allclose(yl, P["yl"], rtol=0, atol=1e-12)
    assert P["yl"].max() > 5.0


def test_quiet_rows_and_unit_ratio_pass_through_bit_exact():
    rate = 16000
    x = (0.01 * np.sin(2 * np.pi * 440 / rate * np.arange(8000))).astype(np.float32)     # -40 dBFS, below the knee
    for kw in ({}, dict(makeup=6.0)):
        y, red = co.compress(x, rate, **kw)
        assert red == 0.0 and np.array_equal(y, co.params(rate, **kw)["m"] * x.astype(np.float64))
        assert np.array_equal(emulate(x, rate, **kw), (F(co.params(rate, **kw)["m"]) * x).astype(F))
    loud = speech_like(0.5, rate, 1)
    y, red = co.compress(loud, rate, ratio=1.0)
    assert red == 0.0 and np.array_equal(y, loud.astype(np.float64))
    assert np.array_equal(emulate(loud, rate, ratio=1.0), loud)


def test_reduction_follows_a_level_step():
    """a step from -40 to -6 dBFS: the reduction settles at (1 - 1/R)(L - T) and reaches it over the attack"""
    rate = 16000
    n = rate
    x = np.full(n, 10 ** (-40 / 20))
    x[n // 2:] = 10 ** (-6 / 20)
    _, red, P = co.compress(x.astype(np.float32), rate, parts=True)
    target = (1 - 1 / 3) * (-6 - -24)
    assert abs(-red - target) < 1e-3
    assert np.all(P["yl"][: n // 2] == 0)
    k = int(np.argmax(P["yl"] > (1 - np.exp(-1)) * target))
    assert abs(k - n // 2 - 5e-3 * rate) <= 2          # one attack time constant (5 ms)


# ---- the tolerance ---------------------------------------------------------------------------------------------------

def worst_emulation(rate, n, names=tuple(PARAMS)):
    worst = 0.0
    for name in names:
        for x in cases(rate, n):
            x = np.asarray(x, F)
            ref, _, P = co.compress(x, rate, parts=True, **PARAMS[name])
            worst = max(worst, error_units(emulate(x, rate, **PARAMS[name]), ref, P))
    return worst


def test_tolerance_has_headroom_over_the_emulation():
    worst = max(worst_emulation(rate, n) for rate, n in ((8000, 4000), (16000, 12000), (48000, 30000)))
    print(f"fp32 emulation {worst:.3f} units (TOL {TOL})")
    assert 4 * worst <= TOL, worst


def test_every_wrong_variant_exceeds_the_tolerance():
    """each variant moves at least one case of the GPU tests past TOL"""
    got = {}
    for kind in VARIANTS:
        for rate, n in ((16000, 12000), (48000, 48000)):
            for name, kw in PARAMS.items():
                for x in cases(rate, n)[:4]:
                    x = np.asarray(x, F)
                    ref, _, P = co.compress(x, rate, parts=True, **kw)
                    got[kind] = max(got.get(kind, 0.0), error_units(variant(x, rate, kind, **kw), ref, P))
    print({k: f"{v:.1f}" for k, v in got.items()})
    for kind in VARIANTS:
        assert got[kind] > TOL, (kind, got[kind])


# ---- spec parsing, the chain order and the CLI -----------------------------------------------------------------------

def test_spec_parsing():
    from viettts_b200.engine import COMPRESSOR_PRESETS, compressor_params
    voice = COMPRESSOR_PRESETS["voice"]
    assert compressor_params("voice", 16000) == voice
    assert list(compressor_params("voice", 16000)) == ["threshold", "ratio", "knee", "attack", "release", "makeup"]
    p = compressor_params("ratio=4, threshold=-30 ,makeup=2.5", 48000)
    assert p == dict(voice, ratio=4.0, threshold=-30.0, makeup=2.5)
    assert list(p) == list(voice)
    assert compressor_params({"knee": 0, "release": 5000}, 8000) == dict(voice, knee=0.0, release=5000.0)
    assert compressor_params("attack=0.7", 16000)["attack"] == float(F(0.7))
    for k, v in compressor_params("threshold=-60,ratio=20,knee=24,attack=200,release=5,makeup=-24", 192000).items():
        assert v == float(F(v))


@pytest.mark.parametrize("spec,rate,key", [("ratio=0.5", 16000, "ratio"), ("threshold=3", 16000, "threshold"),
                                          ("knee=30", 16000, "knee"), ("attack=0.1", 16000, "attack"),
                                          ("release=6000", 16000, "release"), ("makeup=nan", 16000, "makeup"),
                                          ("gain=3", 16000, "gain"), ("ratio=abc", 16000, "ratio"), ("fast", 16000, "fast"),
                                          ({"ratio": float("inf")}, 16000, "ratio"), ("voice", 7999, "rate"),
                                          ("voice", 16000.5, "rate")])
def test_spec_rejections_name_the_key(spec, rate, key):
    from viettts_b200.engine import compressor_params
    with pytest.raises(ValueError, match=key):
        compressor_params(spec, rate)


def test_audio_chain_stage_order():
    from viettts_b200.engine import AudioChain, OptionError
    ch = AudioChain(output_rate=48000, eq="telephone", compress="voice", limit=-1.0, meter=True)
    assert [s[0] for s in ch._stages()] == ["rs", "eq", "cp", "lm", "mt"]
    ch = AudioChain(compress="ratio=2", loudness=-16.0, limit=-1.0)
    assert [s[0] for s in ch._stages()] == ["cp", "lm"]
    assert ch.compress["ratio"] == 2.0
    assert [s[0] for s in AudioChain(compress="voice", denoise=0.5)._stages()] == ["dn", "cp"]
    assert AudioChain().compress is None and [s[0] for s in AudioChain(eq="hp:100")._stages()] == ["eq"]
    with pytest.raises(OptionError) as e:
        AudioChain(compress="ratio=40")
    assert e.value.option == "compress"


@pytest.mark.parametrize("argv", [["--compress", "ratio=0"], ["--compress", "loud"], ["--compress", "attack=1000"],
                                  ["--compress", "knee=x"]])
def test_cli_rejects_bad_compress(argv, capsys):
    from viettts_b200 import synthesizer
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
    assert "--compress" in capsys.readouterr().err
