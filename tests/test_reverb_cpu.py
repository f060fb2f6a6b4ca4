"""CPU: the convolution reverb's float64 definition (oracle/reverb_oracle.py), the synthetic rooms, the error unit and
tolerance the device is held to, the spec parser, the stream's emission count, the AudioChain stage order and the CLI's
argument errors.

Error unit.  The device computes c in fp32 as a partitioned overlap-save convolution: H_k and X_j are FFT-1024s of 512
taps and of the 1024 samples of frame j, each bin summed over k, and block j of c is half of one inverse FFT-1024.  An
fp32 FFT of length N = 2^m errs by at most about m u in the L2 norm (u = 2^-24), so the spectrum error of X_{j-k} H_k is
about 2 m u ||X_{j-k}||_2 ||H_k||_2 and, through the inverse (1/N, Cauchy-Schwarz over the bins, ||X||_2 = sqrt(N)
||x||_2), reaches one output sample as at most about c u ||x over frame j-k||_2 ||h_k||_2 with c = 3 m = 30 for the
two forward transforms, the inverse and the sum.  The mix adds the rounding of y itself and of the dry product:

    unit[t] = 2^-24 (|y64[t]| + (1 - mix) |x[t]| + mix c sum_k ||x over frame j-k||_2 ||h_k||_2),  j = floor(t / 512)

plus, inside the mix term, 2^-40 ||x||_2 ||h||_2: the float64 oracle's own FFT error, which one transform of the whole
row spreads over every sample, silent stretches included (far below fp32's resolution elsewhere).

TOL is at least 4x the worst error of `emulate` (the kernels' algorithm in float32 numpy) over 16, 44.1 and 48 kHz, the
room and hall presets, a 1-tap IR and an IR of 5 r, and every wrong variant exceeds it by orders of magnitude."""
import numpy as np
import pytest
import scipy.fft as sfft

from oracle import reverb_oracle as ro

BLK = 512
C_UNIT = 30.0
TOL = 4.0
RATES = (16000, 44100, 48000)
F32 = np.float32


def cases(rate: int, n: int) -> list:
    """six float32 test rows of n samples: white noise, a gliding tone, tone bursts in silence, clicks, speech-like
    noise bursts under a 4 Hz envelope, and full-scale alternating samples"""
    rng = np.random.default_rng(n + rate)
    t = np.arange(n) / rate
    env = np.clip(np.sin(2 * np.pi * 4 * t), 0, None) ** 2
    clicks = np.zeros(n)
    clicks[::max(1, rate // 7)] = 0.9
    out = [0.3 * rng.standard_normal(n), 0.5 * np.sin(2 * np.pi * (200 * t + 0.5 * 2000 * t * t)),
           np.where((t % 0.25) < 0.05, 0.7 * np.sin(2 * np.pi * 1000 * t), 0.0), clicks, env * 0.5 * rng.standard_normal(n),
           np.where(np.arange(n) % 2 == 0, 1.0, -1.0)]
    return [np.clip(v, -1, 1).astype(F32) for v in out]


def irs(rate: int) -> dict:
    """name -> (ir float32, mix) of the IRs the tolerance is taken over"""
    from viettts_b200.engine import reverb_params
    room, hall = reverb_params("room", rate), reverb_params("hall", rate)
    long_ir = (np.random.default_rng(5).standard_normal(5 * rate) * np.exp(-np.arange(5 * rate) / rate) * 0.02).astype(F32)
    return {"room": (room["ir"], room["mix"]), "hall": (hall["ir"], hall["mix"]), "one_tap": (np.array([0.8], F32), 1.0),
            "five_r": (long_ir, 0.5)}


def emulate(x, h, mix: float, variant: str | None = None) -> np.ndarray:
    """the kernels' algorithm in float32: H_k and X_j by float32 FFT-1024s, block sums in ascending k, the second half of
    the float32 inverse, y = fp32(mix) c + fp32(1 - mix) x.  `variant` names a wrong algorithm (VARIANTS)."""
    x = np.asarray(x, F32)
    h = np.asarray(h, F32)
    if variant == "correlation":
        h = h[::-1].copy()
    n, K = x.size, -(-h.size // BLK)
    if n == 0:
        return np.zeros(0, F32)
    nb = -(-n // BLK)
    xp = np.zeros(BLK * (nb + 1), F32)
    xp[BLK:BLK + n] = x
    X = sfft.rfft(np.lib.stride_tricks.sliding_window_view(xp, 2 * BLK)[::BLK][:nb], axis=1)
    hp = np.zeros((K, 2 * BLK), F32)
    hp[:, :BLK] = np.concatenate([h, np.zeros(K * BLK - h.size, F32)]).reshape(K, BLK)
    H = sfft.rfft(hp, axis=1)
    assert X.dtype == np.complex64 and H.dtype == np.complex64
    shift = 1 if variant == "partition_shift" else 0
    Y = np.zeros((nb, BLK + 1), np.complex64)
    for k in range(min(K, nb)):
        if k + shift < nb:
            Y[k + shift:] += X[:nb - k - shift] * H[k]
    if variant == "bin512":
        Y[:, BLK] = 0
    c = sfft.irfft(Y, n=2 * BLK, axis=1)
    c = (c[:, :BLK] if variant == "half_swapped" else c[:, BLK:]).ravel()[:n]
    wet, dry = F32(mix), F32(1) - F32(mix)
    if variant == "dry_wet":
        wet, dry = dry, wet
    if wet == 0:
        return x.copy()
    return (wet * c + dry * x).astype(F32)


VARIANTS = ("correlation", "partition_shift", "half_swapped", "bin512", "dry_wet")


def unit(ref, x, h, mix: float) -> np.ndarray:
    """the error unit of every output of one row (module docstring)"""
    x = np.asarray(x, F32).astype(np.float64)
    h = np.asarray(h, F32).astype(np.float64)
    n = x.size
    nb, K = -(-n // BLK), -(-h.size // BLK)
    xp = np.zeros(BLK * (nb + 1))
    xp[BLK:BLK + n] = x
    a = np.sqrt(np.sum(np.lib.stride_tricks.sliding_window_view(xp, 2 * BLK)[::BLK][:nb] ** 2, axis=1))
    b = np.sqrt(np.sum(np.concatenate([h, np.zeros(K * BLK - h.size)]).reshape(K, BLK) ** 2, axis=1))
    w = np.convolve(a, b)[:nb]
    m = ro.f32(mix)
    floor = 2.0 ** -16 * np.sqrt(np.sum(x * x) * np.sum(h * h))      # 2^-40 in all: the float64 oracle's own error
    return 2.0 ** -24 * (np.abs(ref) + (1.0 - m) * np.abs(x) + m * (C_UNIT * np.repeat(w, BLK)[:n] + floor))


def error_units(y, ref, x, h, mix: float) -> float:
    err = np.abs(np.asarray(y, np.float64) - ref)
    if not np.any(err):
        return 0.0
    return float(np.max(err / unit(ref, x, h, mix)))


def test_oracle_is_np_convolve():
    rng = np.random.default_rng(1)
    for n, L in ((1, 1), (7, 3), (100, 1), (64, 200), (513, 511), (1000, 1025), (2049, 700)):
        x, h = rng.standard_normal(n), rng.standard_normal(L)
        c = ro.convolve(x, h)
        assert c.shape == (n,)
        assert np.max(np.abs(c - np.convolve(x, h)[:n])) <= 1e-12 * max(1.0, np.max(np.abs(c)))
    x = rng.standard_normal(300).astype(F32)
    h = rng.standard_normal(40).astype(F32)
    y = ro.reverb(x, h, 0.25)
    ref = 0.75 * x.astype(np.float64) + 0.25 * np.convolve(x.astype(np.float64), h.astype(np.float64))[:300]
    assert np.max(np.abs(y - ref)) <= 1e-12
    assert np.array_equal(ro.reverb(x, h, 0.0), x.astype(np.float64))


@pytest.mark.parametrize("rate", [16000, 48000])
@pytest.mark.parametrize("preset", ["room", "hall"])
def test_synthetic_ir(rate, preset):
    from viettts_b200.engine import REVERB_PRESETS, reverb_ir, reverb_params
    p = REVERB_PRESETS[preset]
    h = reverb_params(preset, rate)["ir"]
    d, N = int(np.round(ro.f32(p["predelay"]) * rate / 1000)), int(np.ceil(ro.f32(p["rt60"]) * rate))
    assert h.dtype == np.float32 and h.size == d + N
    assert np.all(h[:d] == 0) and h[d] != 0
    assert abs(np.sum(h.astype(np.float64) ** 2) - 1.0) <= 1e-5
    ref = ro.synthetic_ir(p["rt60"], p["predelay"], 0, rate)
    assert np.array_equal(h, ref.astype(np.float32))
    assert np.array_equal(reverb_ir(ro.f32(p["rt60"]), ro.f32(p["predelay"]), 0, rate), h)
    assert not np.array_equal(reverb_params(dict(p, seed=1), rate)["ir"], h)
    assert np.array_equal(reverb_params(dict(p, seed=0), rate)["ir"], h)
    rt = ro.schroeder_rt60(h, rate)
    assert abs(rt - p["rt60"]) <= 0.1 * p["rt60"], rt


def test_tolerance_has_headroom_over_the_emulation():
    worst = {}
    for rate in RATES:
        for name, (h, mix) in irs(rate).items():
            for i, x in enumerate(cases(rate, rate)):
                if name == "five_r" and i % 2:
                    continue
                ref = ro.reverb(x, h, mix)
                worst[name] = max(worst.get(name, 0.0), error_units(emulate(x, h, mix), ref, x, h, mix))
    print({k: f"{v:.3f}" for k, v in worst.items()})
    assert 4 * max(worst.values()) <= TOL


def test_every_wrong_variant_exceeds_the_tolerance():
    got = {}
    for rate in (16000, 48000):
        for name, (h, mix) in irs(rate).items():
            if name == "five_r":
                continue
            for x in cases(rate, rate // 2)[:2]:
                ref = ro.reverb(x, h, mix)
                for kind in VARIANTS:
                    if kind in ("correlation", "partition_shift") and name == "one_tap":
                        continue          # a single tap is its own reverse; it has one partition
                    if kind == "dry_wet" and mix == 1.0:
                        continue
                    got[kind] = max(got.get(kind, 0.0), error_units(emulate(x, h, mix, kind), ref, x, h, mix))
    print({k: f"{v:.3g}" for k, v in got.items()})
    for kind in VARIANTS:
        assert got[kind] > 100 * TOL, (kind, got[kind])


def test_emulated_mix_zero_is_the_input():
    x = cases(16000, 3000)[0]
    assert np.array_equal(emulate(x, irs(16000)["room"][0], 0.0), x)


# ---- spec parsing, the stream's emission, the chain order and the CLI ------------------------------------------------

def test_spec_parsing():
    from viettts_b200.engine import REVERB_PRESETS, reverb_params
    assert REVERB_PRESETS["room"] == dict(ro.ROOM, seed=0.0) and REVERB_PRESETS["hall"] == dict(ro.HALL, seed=0.0)
    room = reverb_params("room", 16000)
    assert room["mix"] == ro.f32(0.15) and room["seed"] == 0 and room["rt60"] == ro.f32(0.35)
    hall = reverb_params(" HALL ", 48000)
    assert hall["rt60"] == ro.f32(1.8) and hall["predelay"] == 25.0 and hall["mix"] == ro.f32(0.22)
    p = reverb_params("mix=0.4, rt60=1", 16000)
    assert p["mix"] == ro.f32(0.4) and p["rt60"] == 1.0 and p["predelay"] == ro.f32(8.0)
    assert np.array_equal(p["ir"], ro.synthetic_ir(1.0, 8.0, 0, 16000).astype(F32))
    assert reverb_params({"seed": 3, "predelay": 0}, 8000)["ir"][0] != 0
    for spec in ("rt60=0.1,predelay=0,mix=0,seed=0", "rt60=4,predelay=200,mix=1,seed=16777216"):
        for rate in (8000, 192000):
            q = reverb_params(spec, rate)
            assert q["ir"].size <= 5 * rate
    ir = np.array([1.0, -0.5, 0.25], np.float64)
    q = reverb_params({"ir": ir, "mix": 0.5}, 16000)
    assert q["ir"].dtype == np.float32 and np.array_equal(q["ir"], ir.astype(F32)) and q["mix"] == 0.5
    assert reverb_params({"ir": [2.0]}, 16000)["mix"] == room["mix"]                        # not normalized
    assert reverb_params({"ir": np.ones(5 * 8000)}, 8000)["ir"].size == 40000


@pytest.mark.parametrize("spec,rate,key", [("rt60=0.09", 16000, "rt60"), ("rt60=4.1", 16000, "rt60"), ("predelay=-1", 16000, "predelay"),
                                          ("predelay=201", 16000, "predelay"), ("mix=1.01", 16000, "mix"), ("mix=-0.1", 16000, "mix"),
                                          ("mix=nan", 16000, "mix"), ("rt60=nan", 16000, "rt60"), ("seed=-1", 16000, "seed"),
                                          ("seed=1.5", 16000, "seed"), ("seed=nan", 16000, "seed"), ("size=3", 16000, "size"),
                                          ("cathedral", 16000, "cathedral"), ("rt60=x", 16000, "rt60"),
                                          ({"predelay": float("inf")}, 16000, "predelay"), ("room", 7999, "rate"),
                                          ("room", 44100.5, "rate"), ({"ir": [1.0, float("nan")]}, 16000, "ir"),
                                          ({"ir": []}, 16000, "ir"), ({"ir": np.ones(5 * 16000 + 1)}, 16000, "ir"),
                                          ({"ir": [1.0], "mix": float("nan")}, 16000, "mix"), ({"ir": [1.0], "rt60": 1}, 16000, "rt60"),
                                          (3, 16000, "spec")])
def test_spec_rejections_name_the_key(spec, rate, key):
    from viettts_b200.engine import reverb_params
    with pytest.raises(ValueError, match=key):
        reverb_params(spec, rate)


def test_shared_parser_keeps_the_compressor_and_deesser_messages():
    from viettts_b200.engine import compressor_params, deesser_params
    with pytest.raises(ValueError, match=r"^deess: freq=5000 \(the voice preset's\) must lie in \[1000, 3600\] at this rate$"):
        deesser_params("voice", 8000)
    with pytest.raises(ValueError, match=r"^compress: 'loud' is not key=value \(keys threshold, ratio, knee, attack, release, "
                                         r"makeup\) or a preset \(voice\)$"):
        compressor_params("loud", 16000)
    assert compressor_params("ratio=5", 16000)["threshold"] == -24.0


def test_stream_emission_closed_form():
    from viettts_b200.engine import reverb_stream_emitted
    released = 0
    for p in range(3001):
        while BLK * (released // BLK + 1) <= p:          # a block is released once its frame is complete
            released += BLK
        assert reverb_stream_emitted(p) == released == BLK * (p // BLK), p
        assert p - released <= 511
        assert reverb_stream_emitted(p, end=True) == p


def test_audio_chain_stage_order():
    from viettts_b200.engine import AudioChain, OptionError
    ch = AudioChain(output_rate=48000, eq="hs:6000:3", compress="voice", deess="voice", reverb="hall", limit=-1.0, meter=True)
    assert [s[0] for s in ch._stages()] == ["rs", "eq", "cp", "ds", "rv", "lm", "mt"]
    ch = AudioChain(reverb="mix=0.3", loudness=-16.0, limit=-1.0)
    assert [s[0] for s in ch._stages()] == ["rv", "lm"]
    assert [s[0] for s in AudioChain(reverb="room", denoise=0.5, compress="voice")._stages()] == ["dn", "cp", "rv"]
    assert AudioChain().reverb is None and [s[0] for s in AudioChain(deess="voice")._stages()] == ["ds"]
    with pytest.raises(OptionError) as e:
        AudioChain(reverb="rt60=9")
    assert e.value.option == "reverb" and "rt60" in str(e.value)


@pytest.mark.parametrize("argv", [["--reverb", "rt60=9"], ["--reverb", "cave"], ["--reverb", "mix=2"], ["--reverb", "seed=x"],
                                  ["--reverb", "room", "--output-rate", "8001"]])
def test_cli_rejects_bad_reverb(argv, capsys):
    from viettts_b200 import synthesizer
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
    assert "--reverb" in capsys.readouterr().err or "--output-rate" in argv
