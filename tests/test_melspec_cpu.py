"""CPU: the log-mel front end's fp32 arithmetic (oracle/mel_oracle.py `emulate`, csrc/melspec.cu operation for operation)
against the float64 definition on every signal class, the tolerance the GPU tests hold the kernel to, mutations of the
emulation that tolerance must see, and the filterbank span rule.

TOL -- the bound on the error of a log-mel bin in the clipped linear domain, |exp(got) - max(m64, 1e-5)|, in units of
mel_error_scale (2^-24 (log2(1024) ||w x_pair||_2 sum_k fb[m,k] + (1 + |log m_ref|) m_ref), m_ref = max(m64, 1e-5))
-- is pinned against the worst error of the emulation (test_tolerance_has_headroom_over_the_emulation).

Of the mutations, a sign flip of frame B's separated imaginary part alone (bi) would conjugate B[k] and leave |B[k]|
as it is, so no output can show it; the one tested flips the sign of the mirrored bin's imaginary part in B's real
part, which mixes frame A into frame B."""
import numpy as np
import pytest

from oracle import mel_oracle as mo

TOL = 8.0            # mel_error units (see test_tolerance_has_headroom_over_the_emulation)
SR = 16000
BIN_HZ = SR / 1024


def _tone(f, S, rng, amp=0.5):
    return amp * np.sin(2 * np.pi * f / SR * np.arange(S) + rng.uniform(0, 2 * np.pi))


def _noise(B, S, rng):
    return 0.1 * rng.standard_normal((B, S))


def _tones_on_bin(B, S, rng):
    return np.stack([_tone(round(f / BIN_HZ) * BIN_HZ, S, rng) for f in (100.0, 1000.0, 7900.0)][:B])


def _tones_half_bin(B, S, rng):
    return np.stack([_tone((np.floor(f / BIN_HZ) + 0.5) * BIN_HZ, S, rng) for f in (100.0, 1000.0, 7900.0)][:B])


def _chirp(B, S, rng):
    t = np.arange(S) / SR
    T = S / SR
    return np.stack([(0.3 + 0.3 * b) * np.sin(np.pi * 8000.0 / T * t ** 2 + rng.uniform(0, 2 * np.pi)) for b in range(B)])


def _dc(B, S, rng):
    return np.stack([np.full(S, v) for v in (0.5, -0.999, 1e-3)][:B])


def _clicks(B, S, rng):
    """unit clicks on the first and last samples, on hop boundaries (256 k and 256 k - 1) and on each frame's edge"""
    x = np.zeros((B, S))
    x[0, 0], x[0, -1] = 1.0, -1.0
    x[1, 256 :: 256] = 0.7
    x[1, 255 :: 256] = -0.7
    x[2, 128 :: 512] = 1.0
    x[2, min(S - 1, 383)] = -1.0
    return x[:B]


def _int16_square(B, S, rng):
    """full-scale int16 square waves (+32767 / -32768) read as wav / 32768, at three periods"""
    n = np.arange(S)
    return np.stack([np.where((n // p) % 2 == 0, 32767, -32768) / 32768.0 for p in (80, 33, 2)][:B])


def _zeros(B, S, rng):
    return np.zeros((B, S))


def _tiny(B, S, rng):
    """1e-6 amplitude: the magnitudes sit at the sqrt(1e-9) floor and the mel sums at the 1e-5 clip"""
    return 1e-6 * np.stack([_tone(1000.0, S, rng, 1.0), rng.standard_normal(S), _tone(250.0, S, rng, 1.0) + rng.standard_normal(S)][:B])


SIGNALS = {"noise": _noise, "tones_on_bin": _tones_on_bin, "tones_half_bin": _tones_half_bin, "chirp": _chirp, "dc": _dc,
           "clicks": _clicks, "int16_square": _int16_square, "zeros": _zeros, "tiny": _tiny}


def signal(name, B, S, seed=0):
    return SIGNALS[name](B, S, np.random.default_rng([seed, S])).astype(np.float32)


def three_minutes(seed=0):
    """one 3-minute row: speech-band noise bursts between tones, with silent gaps"""
    rng = np.random.default_rng(seed)
    S = 180 * SR
    x = 0.05 * rng.standard_normal(S) * (np.sin(2 * np.pi * 0.5 * np.arange(S) / SR) > 0)
    x += _tone(440.0, S, rng, 0.2) + _tone(3000.0, S, rng, 0.05)
    x[S // 3 : S // 3 + 5 * SR] = 0.0
    return x[None].astype(np.float32)


def banks():
    """the default Slaney bank, fmin 80 / fmax 7600, the sr = 22050 bank, and the default with an all-zero row and a
    row with interior zeros"""
    from viettts_b200.weights import mel_filterbank
    holed = mel_filterbank().copy()
    holed[7] = 0.0
    lo, hi = mo.mel_spans(holed[40:41])
    holed[40, lo[0] + 1 : hi[0] - 1 : 2] = 0.0
    return {"default": mel_filterbank(), "fmin80_fmax7600": mel_filterbank(16000, 1024, 80, 80.0, 7600.0),
            "sr22050": mel_filterbank(22050, 1024, 80, 0.0, 11025.0), "holed": holed}


def error_units(got, y, fb):
    units, bad_clip = mo.mel_error(got, y, fb, TOL)
    return float(units.max()), bad_clip


# ---- the emulation against float64 ----------------------------------------------------------------------------------

EMULATION_S = (512, 768, 1024, 1280, 4608)


def _emulated_worst():
    fb = banks()["default"]
    worst = {}
    for name in SIGNALS:
        for S in EMULATION_S:
            y = signal(name, 3, S)
            e, bad = error_units(mo.emulate(y, fb), y, fb)
            assert bad == 0, (name, S)
            worst[name] = max(worst.get(name, 0.0), e)
    return worst


@pytest.mark.parametrize("name", list(SIGNALS))
def test_emulation_within_tolerance(name):
    fb = banks()["default"]
    worst = 0.0
    for S in EMULATION_S:
        y = signal(name, 3, S)
        got = mo.emulate(y, fb)
        e, bad = error_units(got, y, fb)
        assert bad == 0, S
        worst = max(worst, e)
    print(f"{name}: {worst:.3f} units")
    assert worst <= TOL / 3


@pytest.mark.parametrize("bank", ["fmin80_fmax7600", "sr22050", "holed"])
def test_emulation_within_tolerance_other_banks(bank):
    fb = banks()[bank]
    worst = 0.0
    for name in ("noise", "chirp", "tones_half_bin", "tiny"):
        y = signal(name, 3, 1280, seed=1)
        e, bad = error_units(mo.emulate(y, fb), y, fb)
        assert bad == 0, name
        worst = max(worst, e)
    print(f"{bank}: {worst:.3f} units")
    assert worst <= TOL / 3


def test_three_minute_row_emulation():
    fb = banks()["default"]
    y = three_minutes()
    e, bad = error_units(mo.emulate(y, fb), y, fb)
    print(f"3 min: {e:.3f} units")
    assert bad == 0 and e <= TOL / 3


def test_clipped_bins_are_the_clip_bit_for_bit():
    fb = banks()["default"]
    for name in ("zeros", "tiny"):
        y = signal(name, 3, 1024)
        got = mo.emulate(y, fb)
        m64 = mo.mel_linear(y, dtype=np.float64, fb=fb)
        assert (m64 < 1e-5).any()
        assert np.all(got[m64 < 0.5e-5] == mo.LOG_CLIP), name
    assert np.all(mo.emulate(signal("zeros", 3, 512), fb) == mo.LOG_CLIP)


def test_tolerance_has_headroom_over_the_emulation():
    worst = _emulated_worst()
    w = max(worst.values())
    print("fp32 emulation, worst units per class: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    print(f"worst {w:.3f} units, TOL {TOL}, margin {TOL / w:.1f}x")
    assert 3 * w <= TOL <= 10 * w, w


# ---- mutations the tolerance must see ---------------------------------------------------------------------------

@pytest.mark.parametrize("mutation", [{"pad": "symmetric"}, {"drop_last_bin": True}, {"b_mirror_sign": True},
                                      {"chain_extra_step": True}], ids=["symmetric_pad", "span_short", "b_mirror_sign", "chain_long"])
def test_mutations_exceed_tolerance(mutation):
    fb = banks()["default"]
    worst = 0.0
    for name in ("noise", "chirp", "clicks", "tones_half_bin"):
        for S in (512, 768):
            y = signal(name, 3, S)
            worst = max(worst, error_units(mo.emulate(y, fb, **mutation), y, fb)[0])
    print(f"{mutation}: {worst:.3g} units")
    assert worst > TOL


# ---- the filterbank span rule -----------------------------------------------------------------------------------

@pytest.mark.parametrize("bank", ["default", "fmin80_fmax7600", "sr22050", "holed"])
def test_spans_cover_every_nonzero_weight(bank):
    fb = banks()[bank]
    lo, hi = mo.mel_spans(fb)
    k = np.arange(fb.shape[1])
    outside = (k[None, :] < lo[:, None]) | (k[None, :] >= hi[:, None])
    assert np.all(fb[outside] == 0)
    live = hi > lo
    rows = np.flatnonzero(live)
    assert np.all(fb[rows, lo[live]] != 0) and np.all(fb[rows, hi[live] - 1] != 0)
    assert np.all((lo[~live] == 0) & (hi[~live] == 0))
    assert np.all((0 <= lo) & (lo <= hi) & (hi <= fb.shape[1]))
    if bank == "holed":
        assert not live[7] and hi[40] - lo[40] > np.count_nonzero(fb[40])


def test_span_sum_equals_the_dense_product():
    """summing each row over its span gives the float64 dense product, interior zeros included"""
    fb = banks()["holed"]
    lo, hi = mo.mel_spans(fb)
    mag = np.random.default_rng(4).random((5, fb.shape[1]))
    dense = mag @ fb.astype(np.float64).T
    spans = np.stack([mag[:, lo[m] : hi[m]] @ fb[m, lo[m] : hi[m]].astype(np.float64) for m in range(len(fb))], 1)
    assert np.allclose(spans, dense, rtol=1e-12, atol=0)


def test_error_scale_uses_the_pair_norm():
    """a silent frame packed with a loud one is held to the loud one's round-off, a silent pair to the clip alone"""
    fb = banks()["default"]
    y = np.zeros((1, 2048), np.float32)
    y[0, 1152:] = 0.5                      # frame f reads [256 f - 384, 256 f + 640): frames 0..2 silent, 3.. loud
    scale, _ = mo.mel_error_scale(y, fb)
    assert np.all(scale[0, :2] == 2.0 ** -24 * (1 - np.log(1e-5)) * 1e-5)
    assert scale[0, 2].min() > 1e3 * scale[0, 0].max()
