"""CPU: the bed's definition (oracle/bed_oracle.py), the tolerance the GPU tests hold the device to, the spec parser, the
pink preset, the AudioChain stage order and the CLI's --bed parsing and stereo downmix.

TOL bounds error_units(y), the per-sample error of y = x + g e bl against float64 in units of

    u[t] = 2^-24 (3 |y64| + |g e bl|64 (3 + (ln 10 / 20) Lam (1 + sqrt(1 / (1 - a_R)) + sqrt(1 / (1 - a_A))))
                  + 2 g (|bl| + e bw)),

the de-esser's unit (tests/test_deesser_cpu.py) with the detector's gain acting on the bed term g e bl instead of on the
high band: an error of e dB in y_L moves y by (ln 10 / 20) e |g e bl|, the 3 |y64| covers the rounding of fmaf(g e, bl,
x), and the 3 exp10f and the product g e.  The envelope and the crossfade weights come from cospif / sinpif, whose error
is a few 2^-24 of 1, not of the weight (1 - cos near a fade's start cancels): the last term charges that absolute
error to g |bl| for the envelope and to g e bw for the weights, bw = |b[u]| (+ |b[P + u]| over the crossfade).  TOL is
pinned against an fp32 numpy emulation of the kernels (the compressor's block scans on the key row, then the apply),
and every wrong variant in `VARIANTS` exceeds it."""
import struct

import numpy as np
import pytest

from oracle import bed_oracle as bo
from oracle import compressor_oracle as co
from test_compressor_cpu import consts, fma, speech_like
from test_deesser_cpu import detector32

TOL = 4.0            # error_units (see test_tolerance_has_headroom_over_the_emulation)
F = np.float32

PARAMS = {
    "default": {},
    "deep": dict(duck=40.0, threshold=-50.0),
    "fast": dict(attack=0.5, release=5.0, threshold=-30.0),
    "slow": dict(attack=200.0, release=5000.0, duck=6.0),
}


def shape(rate, Fi=0.25, Tt=0.3, C=0.05, o=0.1):
    """the sample counts of the GPU tests' shapes: fade-in, tail, crossfade, offset in seconds"""
    return dict(Fi=int(round(Fi * rate)), Tt=int(round(Tt * rate)), C=int(round(C * rate)), o=int(round(o * rate)))


def short_bed(rate, seconds=0.6, seed=1):
    """a pink bed at -30 dBFS RMS, shorter than the rows: it wraps several times"""
    from viettts_b200.engine import pink_bed
    return (10 ** (-30 / 20) * pink_bed(seed, seconds, rate)).astype(F)


def cases(rate, n):
    return [speech_like(n / rate + 0.01, rate, 3)[:n], (0.3 * np.sin(2 * np.pi * 200 / rate * np.arange(n))).astype(F),
            np.zeros(n, F)]


# ---- fp32 emulation of bed.cu ----------------------------------------------------------------------------------------

def emulate(x, b, rate, Fi=0, Tt=0, C=0, o=0, **kw):
    """y of bed.cu's one-shot arithmetic in fp32 numpy"""
    p = bo.params(rate, **kw)
    x = np.asarray(x, F)
    n = x.size
    key = np.concatenate([x, np.zeros(Tt, F)])
    if key.size == 0:
        return key
    ylc = np.minimum(detector32(key, consts(p)), F(p["duck"]))
    g = np.where(ylc > 0, np.power(F(10), (-ylc / F(20)).astype(F)), F(1)).astype(F)
    t = np.arange(n + Tt)
    e = np.ones(n + Tt, F)
    if Fi > 0:
        m = t < Fi
        e[m] = (F(0.5) - F(0.5) * np.cos(F(np.pi) * (t[m].astype(F) / F(Fi))).astype(F)).astype(F)
    if Tt > 0:
        m = t >= n
        e[m] = (e[m] * (F(0.5) + F(0.5) * np.cos(F(np.pi) * ((t[m] - n + 1).astype(F) / F(Tt))).astype(F))).astype(F)
    b = np.asarray(b, F)
    P = b.size - C
    u = (t + o) % P
    bl = b[u].copy()
    if C > 0:
        m = u < C
        w = (u[m].astype(F) / F(2 * C)).astype(F)
        s, c = np.sin(F(np.pi) * w).astype(F), np.cos(F(np.pi) * w).astype(F)
        bl[m] = fma(s, b[u[m]], (c * b[P + u[m]]).astype(F))
    return fma((g * e).astype(F), bl, key)


def error_units(y, ref, P):
    """max |y - ref| / u[t] over the row (see the module docstring); P the oracle's parts"""
    y = np.asarray(y, np.float64)
    if y.size == 0:
        return 0.0
    L = P["L"]
    above = np.isfinite(L) & (L >= P["threshold"] - P["knee"] / 2)
    lam = float(np.abs(L[above]).max()) if above.any() else 0.0
    k = np.log(10) / 20 * lam * (1 + np.sqrt(1 / (1 - P["aR"])) + np.sqrt(1 / (1 - P["aA"])))
    u = 2.0 ** -24 * (3 * np.abs(ref) + np.abs(P["g"] * P["e"] * P["bl"]) * (3 + k) + 2 * P["g"] * (np.abs(P["bl"]) + P["e"] * P["bw"]))
    err = np.abs(y - ref)
    if np.any((u == 0) & (err > 0)):
        return np.inf
    return float(np.max(np.where(u > 0, err / np.where(u > 0, u, 1), 0.0)))


# ---- wrong variants of the definition (float64) ----------------------------------------------------------------------

def variant(x, b, rate, kind, Fi=0, Tt=0, C=0, o=0, **kw):
    """y of the oracle with one deliberate mistake"""
    ref, _, P = bo.mix(x, b, rate, Fi, Tt, C, o, parts=True, **kw)
    n = len(x)
    g, e, bl = P["g"], P["e"], P["bl"]
    if kind == "noseam":
        bl = np.asarray(b, F).astype(np.float64)[(np.arange(n + Tt) + o) % (len(b) - C)]
    elif kind == "nocap":
        g = 10.0 ** (-P["yl"] / 20.0)
    elif kind == "swap":
        yl = co.attack(co.release(P["xl"], P["aA"], P["bA"]), P["aR"], P["bR"])
        g = 10.0 ** (-np.minimum(yl, P["duck"]) / 20.0)
    elif kind == "nofadeout":
        e = bo.envelope(n, Fi, 0)
        e = np.concatenate([e, np.ones(Tt)])
    elif kind == "linear":
        t = np.arange(n + Tt)
        u = (t + o) % (len(b) - C)
        m = u < C
        b64 = np.asarray(b, F).astype(np.float64)
        bl = bl.copy()
        bl[m] = (u[m] / C) * b64[u[m]] + (1 - u[m] / C) * b64[len(b) - C + u[m]]
    return P["key"] + g * e * bl


VARIANTS = ("noseam", "nocap", "swap", "nofadeout", "linear")


# ---- the definition --------------------------------------------------------------------------------------------------

def test_duck_zero_is_the_plain_sum():
    rate = 16000
    x, b, s = speech_like(1.0, rate, 2), short_bed(rate), shape(rate)
    y, red, P = bo.mix(x, b, rate, **s, duck=0.0, parts=True)
    assert red == 0.0 and np.all(P["g"] == 1.0)
    key = np.concatenate([x.astype(np.float64), np.zeros(s["Tt"])])
    assert np.array_equal(y, key + P["e"] * P["bl"])


def test_silent_key_gives_the_bed_under_its_envelopes():
    rate = 16000
    b, s = short_bed(rate), shape(rate)
    x = np.zeros(rate, F)
    y, red = bo.mix(x, b, rate, **s)
    assert red == 0.0
    assert np.array_equal(y, bo.envelope(rate, s["Fi"], s["Tt"]) * bo.looped(b, rate + s["Tt"], s["C"], s["o"]))


def test_seam_is_continuous():
    rate = 16000
    C = 800
    b = np.cos(2 * np.pi * 3 * np.arange(8000) / 8000).astype(F)      # smooth, and its end meets its start
    P = b.size - C
    bl = bo.looped(b, 3 * P, C, 0)
    assert bl[C] == b[C] and abs(bl[C - 1] - b[C - 1]) < 0.02         # at u = C: the crossfade ends on b[C]
    assert bl[P - 1] == b[P - 1] and abs(bl[P] - b[P]) < 1e-12         # the wrap: b[P - 1] is followed by b[P]
    assert np.max(np.abs(np.diff(bl))) < 3 * np.max(np.abs(np.diff(b)))
    w = np.arange(C) / (2.0 * C)
    assert np.allclose(np.sin(np.pi * w) ** 2 + np.cos(np.pi * w) ** 2, 1.0)   # equal power


def test_tail_is_exactly_tt_and_ends_at_zero():
    rate = 16000
    x, b, s = speech_like(0.5, rate, 4), short_bed(rate), shape(rate)
    y, _, P = bo.mix(x, b, rate, **s, parts=True)
    n = x.size
    assert y.size == n + s["Tt"] and P["e"][-1] == 0.0 and y[-1] == 0.0
    assert np.all(np.diff(P["e"][n:]) <= 0) and P["e"][n] > 0.99
    assert np.all(np.diff(P["y1"][n:]) < 0) and P["yl"][-1] < P["yl"][n:].max()   # the detector releases over the tail
    assert bo.mix(x, b, rate, **dict(s, Tt=0))[0].size == n


def test_no_bed_is_the_identity():
    x = speech_like(0.3, 16000, 5)
    y, red = bo.mix(x, None, 16000, **shape(16000))
    assert red == 0.0 and np.array_equal(y, x.astype(np.float64))


def test_ducks_under_the_voice_by_at_most_the_depth():
    rate = 16000
    x, b, s = speech_like(2.0, rate, 6), short_bed(rate), shape(rate)
    y, red, P = bo.mix(x, b, rate, **s, duck=12.0, parts=True)
    assert -12.0 <= red < -10.0 and P["ylc"].max() <= 12.0


# ---- the tolerance ---------------------------------------------------------------------------------------------------

def worst_emulation(rate, n):
    worst = 0.0
    b, s = short_bed(rate), shape(rate)
    for kw in PARAMS.values():
        for x in cases(rate, n):
            ref, _, P = bo.mix(x, b, rate, **s, parts=True, **kw)
            worst = max(worst, error_units(emulate(x, b, rate, **s, **kw), ref, P))
    return worst


def test_tolerance_has_headroom_over_the_emulation():
    worst = max(worst_emulation(rate, n) for rate, n in ((16000, 12000), (44100, 20000), (48000, 30000)))
    print(f"fp32 emulation {worst:.3f} units (TOL {TOL})")
    assert 4 * worst <= TOL, worst


def test_every_wrong_variant_exceeds_the_tolerance():
    got = {}
    for rate, n in ((16000, 16000), (48000, 40000)):
        b, s = short_bed(rate), shape(rate)
        for kw in PARAMS.values():
            for x in cases(rate, n)[:2]:
                ref, _, P = bo.mix(x, b, rate, **s, parts=True, **kw)
                for kind in VARIANTS:
                    got[kind] = max(got.get(kind, 0.0), error_units(variant(x, b, rate, kind, **s, **kw), ref, P))
    print({k: f"{v:.1f}" for k, v in got.items()})
    for kind in VARIANTS:
        assert got[kind] > TOL, (kind, got[kind])


# ---- spec parsing, the pink preset, the chain order and the CLI ------------------------------------------------------

def test_spec_parsing():
    from viettts_b200.engine import BED_DEFAULTS, bed_params, bed_specs
    assert {k: BED_DEFAULTS[k] for k in bo.DEFAULTS} == bo.DEFAULTS
    p = bed_params("pink", 16000)
    assert {k: p[k] for k in BED_DEFAULTS} == BED_DEFAULTS
    assert (p["Nb"], p["Fi"], p["Tt"], p["C"], p["o"], p["audio_rate"], p["seed"]) == (128000, 4000, 16000, 800, 0, 16000, 0)
    p = bed_params("pink, duck=20 ,seed=7,length=2,offset=1.5,tail=0", 48000)
    assert (p["duck"], p["seed"], p["Nb"], p["o"], p["Tt"]) == (20.0, 7, 96000, 72000, 0)
    a = np.random.default_rng(0).standard_normal(22050).astype(F)
    p = bed_params({"audio": a, "audio_rate": 22050, "level": -20, "xfade": 10}, 16000)
    assert p["Nb"] == 16000 and p["level"] == -20.0 and p["C"] == 160 and np.array_equal(p["audio"], a)
    assert bed_params({"audio": a[:16000]}, 16000)["audio_rate"] == 16000
    ps = bed_specs(["pink", "pink,seed=3,level=-40", {"audio": a, "audio_rate": 22050}], 16000)
    assert len(ps) == 3 and ps[1]["level"] == -40.0


@pytest.mark.parametrize("spec,rate,key", [("pink,level=-5", 16000, "level"), ("pink,level=-61", 16000, "level"),
                                          ("pink,duck=41", 16000, "duck"), ("pink,duck=-1", 16000, "duck"),
                                          ("pink,threshold=1", 16000, "threshold"), ("pink,attack=0.1", 16000, "attack"),
                                          ("pink,release=6000", 16000, "release"), ("pink,fade_in=5001", 16000, "fade_in"),
                                          ("pink,tail=10001", 16000, "tail"), ("pink,tail=-1", 16000, "tail"),
                                          ("pink,xfade=1001", 16000, "xfade"), ("pink,length=0.6,xfade=300", 16000, "xfade"),
                                          ("pink,offset=8", 16000, "offset"), ("pink,offset=-1", 16000, "offset"),
                                          ("pink,seed=1.5", 16000, "seed"), ("pink,length=0.4", 16000, "length"),
                                          ("pink,length=601", 16000, "length"), ("pink,duck=nan", 16000, "duck"),
                                          ("pink,loud=3", 16000, "loud"), ("pink,duck", 16000, "duck"),
                                          ("music", 16000, "pink"), ("pink", 7999, "rate"), ("pink", 11025, "rate"),
                                          ({"audio": np.zeros(7999)}, 16000, "lasts"),
                                          ({"audio": np.zeros(16000), "seed": 1}, 16000, "seed"),
                                          ({"audio": np.zeros((2, 16000))}, 16000, "mono"),
                                          ({"audio": np.full(16000, np.inf)}, 16000, "finite"),
                                          ({"audio": np.zeros(16000), "audio_rate": 0}, 16000, "audio_rate"),
                                          ({"audio": np.zeros(16000), "audio_rate": 16001}, 16000, "1024"),
                                          ({"audio_rate": 8000}, 16000, "audio_rate"), (3, 16000, "string or a dict")])
def test_spec_rejections_name_the_key(spec, rate, key):
    from viettts_b200.engine import bed_params
    with pytest.raises(ValueError, match=key):
        bed_params(spec, rate)


def test_bank_rejections():
    from viettts_b200.engine import BedBank, bed_specs
    with pytest.raises(ValueError, match="duck"):
        bed_specs(["pink", "pink,duck=3"], 16000)
    with pytest.raises(ValueError, match="1 to 8"):
        bed_specs(["pink"] * 9, 16000)
    with pytest.raises(ValueError, match="xfade"):
        bed_specs(["pink,xfade=200", {"audio": np.zeros(8000)}], 16000)
    bank = BedBank(None, np.zeros(2, np.int64), np.zeros(2, np.int32), bed_specs(["pink", "pink,seed=1"], 16000), 16000)
    assert bank.index(1, 3).tolist() == [1, 1, 1] and bank.index([-1, 0, 1], 3).tolist() == [-1, 0, 1]
    for bad in (2, -2, 0.5, [0, 1]):
        with pytest.raises(ValueError, match="bed index"):
            bank.index(bad, 3)


def test_pink_preset_is_deterministic_per_seed():
    from viettts_b200.engine import bed_params, pink_bed
    a, b, c = pink_bed(3, 1.0, 16000), pink_bed(3, 1.0, 16000), pink_bed(4, 1.0, 16000)
    assert a.dtype == F and a.size == 16000 and np.array_equal(a, b) and not np.array_equal(a, c)
    assert abs(np.sqrt(np.mean(a.astype(np.float64) ** 2)) - 1) < 1e-6
    spec = np.abs(np.fft.rfft(a.astype(np.float64))) ** 2                 # 1/f: about 3 dB per octave down
    lo, hi = spec[100:200].mean(), spec[1600:3200].mean()
    assert 10 < 10 * np.log10(lo / hi) < 14
    assert np.array_equal(bed_params("pink,seed=3,length=1", 16000)["audio"], a)


def test_audio_chain_stage_order():
    from viettts_b200.engine import AudioChain, OptionError
    ch = AudioChain(output_rate=48000, compress="voice", reverb="room", bed="pink", limit=-1.0, meter=True)
    assert [s[0] for s in ch._stages()] == ["rs", "cp", "rv", "bd", "lm", "mt"]
    ch = AudioChain(bed="pink,duck=6", loudness=-16.0, encoding="ulaw")
    assert [s[0] for s in ch._stages()] == ["bd", "lm"] and ch.bed[0]["duck"] == 6.0
    assert AudioChain().bed is None
    with pytest.raises(OptionError) as e:
        AudioChain(bed="pink,duck=50")
    assert e.value.option == "bed" and "duck" in str(e.value)
    with pytest.raises(OptionError) as e:
        AudioChain(bed="pink", output_rate=11025)
    assert e.value.option == "bed"


def wav_bytes(codes, rate, channels):
    data = np.asarray(codes, "<i2").tobytes()
    fmt = struct.pack("<IHHIIHH", 16, 1, channels, rate, rate * 2 * channels, 2 * channels, 16)
    chunks = b"fmt " + fmt + b"data" + struct.pack("<I", len(data)) + data
    return b"RIFF" + struct.pack("<I", 4 + len(chunks)) + b"WAVE" + chunks


def test_stereo_wav_downmix(tmp_path):
    from viettts_b200 import synthesizer
    rng = np.random.default_rng(0)
    lr = rng.integers(-32768, 32768, (5000, 2)).astype(np.int16)
    (tmp_path / "s.wav").write_bytes(wav_bytes(lr.reshape(-1), 22050, 2))
    with pytest.raises(ValueError, match="2 channels"):
        synthesizer.read_wav_codes(tmp_path / "s.wav")                   # mono readers still refuse it
    codes, rate, enc = synthesizer.read_wav_codes(tmp_path / "s.wav", stereo=True)
    assert (rate, enc) == (22050, "pcm16") and np.array_equal(codes, lr)
    v, rate = synthesizer.read_bed_wav(tmp_path / "s.wav")
    assert rate == 22050 and v.dtype == F
    assert np.array_equal(v, ((lr[:, 0].astype(np.float64) + lr[:, 1]) / 2 / 32767).astype(F))
    synthesizer.write_wav(tmp_path / "m.wav", v, 22050)
    m, _ = synthesizer.read_bed_wav(tmp_path / "m.wav")
    assert np.array_equal(m, synthesizer.float_to_pcm16(v).astype(F) / F(32767))


def test_cli_bed_argument(tmp_path):
    from viettts_b200 import synthesizer
    assert synthesizer.bed_arg("pink,seed=2,duck=6") == "pink,seed=2,duck=6"
    lr = np.tile(np.array([[1000, -3000]], np.int16), (30000, 1))
    (tmp_path / "b.wav").write_bytes(wav_bytes(lr.reshape(-1), 44100, 2))
    spec = synthesizer.bed_arg(f"{tmp_path / 'b.wav'},level=-24,offset=0.2")
    assert spec["audio_rate"] == 44100 and spec["level"] == "-24" and spec["offset"] == "0.2"
    assert np.all(spec["audio"] == F(-1000 / 32767))
    from viettts_b200.engine import AudioChain
    assert AudioChain(bed=spec, output_rate=48000).bed[0]["Nb"] == 32654        # ceil(30000 * 160 / 147)


@pytest.mark.parametrize("argv", [["--bed", "pink,duck=50"], ["--bed", "music"], ["--bed", "/nonexistent/bed.wav"],
                                  ["--bed", "pink,level"], ["--bed", "pink", "--output-rate", "11025"]])
def test_cli_rejects_bad_bed(argv, capsys):
    from viettts_b200 import synthesizer
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
    assert "--bed" in capsys.readouterr().err
