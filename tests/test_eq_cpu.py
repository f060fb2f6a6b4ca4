"""CPU: the equalizer's designer (vtts_eq_design against scipy and the oracle's formulas), the state-variable form of
every section (oracle/eq_oracle.py svf_params), the tolerance the GPU tests hold the device to, the stream's invariance
to push patterns, spec parsing, the Engine validators and the CLI's argument errors.

TOL -- the bound on error_units(y), the error of y against float64 in units of 2^-24 max |x| ||h||_1 (||h||_1 bounds
the output of the cascade for |x| <= max |x|) -- is pinned against an fp32 numpy emulation of eq.cu's arithmetic: the
per-section lane segments, their scans, the block chain and the output pass."""
import numpy as np
import pytest
from scipy import signal

from oracle import eq_oracle as eo

TOL = 96.0           # error_units (see test_tolerance_has_headroom_over_the_emulation)

VOICE = "hp:80:4,ls:200:-2,pk:3000:1:3,hs:6000:2"
WORST = "hp:60:8,lp:7000:8"


def elliptic_hp(rate):
    return signal.ellip(6, 0.5, 60, 80, "highpass", fs=rate, output="sos")


def lib():
    from viettts_b200 import _lib, build
    build.build()
    return _lib.load()


def design(kind, rate, f0, q=1.0, gain=0.0, order=2):
    import ctypes
    sos = np.zeros((8, 6))
    k = ctypes.c_int()
    rc = lib().vtts_eq_design(kind, rate, f0, q, gain, order, sos.ctypes.data, ctypes.byref(k))
    return rc, sos[:k.value]


def error_units(y, ref, x, sos):
    scale = float(np.abs(np.asarray(x, np.float64)).max()) * eo.impulse_l1(sos) * 2.0 ** -24
    err = float(np.abs(np.asarray(y, np.float64) - ref).max())
    return 0.0 if err == 0 else err / scale


def tone(f, n, rate, amp=0.9):
    return amp * np.sin(2 * np.pi * f / rate * np.arange(n))


def clicks(n):
    x = np.zeros(n)
    x[n // 5] = 1.0
    x[n // 2] = -1.0
    x[n // 2 + 7] = 0.8
    return x


def noise(n, seed=0):
    return np.clip(np.random.default_rng(seed).standard_normal(n) / 3, -1, 1)


# ---- designer ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("btype,kind", [("highpass", eo.HIGHPASS), ("lowpass", eo.LOWPASS)])
@pytest.mark.parametrize("order", range(1, 9))
@pytest.mark.parametrize("rate,f0", [(8000, 300.0), (16000, 60.0), (48000, 3400.0), (192000, 200.0), (44100, 0.45 * 44100)])
def test_butterworth_equals_scipy(btype, kind, order, rate, f0):
    rc, sos = design(kind, rate, f0, order=order)
    assert rc == 0 and sos.shape == (-(-order // 2), 6) and np.all(sos[:, 3] == 1.0)
    ref = eo.butter(btype, order, f0, rate)
    # 16384 frequencies from 10 Hz (the designer's lowest f0) to Nyquist
    w = np.linspace(2 * np.pi * 10 / rate, np.pi, 16385)[:-1]
    h = signal.sosfreqz(sos, w)[1]
    h_ref = signal.sosfreqz(ref, w)[1]
    # in dB wherever the response is above -40 dB; deeper in the stopband the double coefficients themselves carry a
    # relative error of eps / |1 + a1 z^-1 + a2 z^-2| (near DC a high-pass numerator (1 - z^-1)^2 cancels to eps / w^2),
    # so there the responses are compared absolutely
    db, db_ref = 20 * np.log10(np.abs(h)), 20 * np.log10(np.abs(h_ref))
    band = db_ref > -40
    assert np.abs(db - db_ref)[band].max() <= 1e-9
    assert np.abs(h - h_ref).max() <= 1e-10


@pytest.mark.parametrize("rate", [8000, 16000, 44100, 48000, 192000])
def test_rbj_kinds_equal_the_oracle(rate):
    for f0 in (10.0, 200.0, 3000.0, 0.45 * rate):
        for gain in (-24.0, -2.0, 0.0, 3.0, 24.0):
            for S in (0.1, 0.5, 1.0):
                assert np.abs(design(eo.LOWSHELF, rate, f0, S, gain)[1] - eo.shelf(False, f0, gain, S, rate)).max() <= 1e-12
                assert np.abs(design(eo.HIGHSHELF, rate, f0, S, gain)[1] - eo.shelf(True, f0, gain, S, rate)).max() <= 1e-12
            for q in (0.1, 0.707, 30.0):
                assert np.abs(design(eo.PEAKING, rate, f0, q, gain)[1] - eo.peaking(f0, q, gain, rate)).max() <= 1e-12
        for q in (0.1, 10.0, 30.0):
            assert np.abs(design(eo.NOTCH, rate, f0, q)[1] - eo.notch(f0, q, rate)).max() <= 1e-12


@pytest.mark.parametrize("args", [(eo.HIGHPASS, 7999, 100.0), (eo.HIGHPASS, 192001, 100.0), (eo.LOWPASS, 16000, 9.9),
                                  (eo.LOWPASS, 16000, 7200.1), (eo.HIGHPASS, 16000, 100.0, 1.0, 0.0, 0),
                                  (eo.HIGHPASS, 16000, 100.0, 1.0, 0.0, 9), (eo.PEAKING, 16000, 100.0, 0.09, 3.0),
                                  (eo.PEAKING, 16000, 100.0, 31.0, 3.0), (eo.PEAKING, 16000, 100.0, 1.0, 24.5),
                                  (eo.LOWSHELF, 16000, 100.0, 0.0, 3.0), (eo.HIGHSHELF, 16000, 100.0, 1.1, 3.0),
                                  (eo.NOTCH, 16000, 100.0, 0.05), (6, 16000, 100.0), (-1, 16000, 100.0),
                                  (eo.LOWPASS, 16000, float("nan")), (eo.PEAKING, 16000, 100.0, 1.0, float("nan"))])
def test_designer_rejects_out_of_range(args):
    assert design(*args)[0] == -1


def test_designs_are_valid_filters():
    for rate in (8000, 48000, 192000):
        for kind in range(6):
            for f0 in (10.0, 0.45 * rate):
                rc, sos = design(kind, rate, f0, 1.0 if kind in (eo.LOWSHELF, eo.HIGHSHELF) else 30.0, 24.0, 8)
                assert rc == 0 and eo.valid(sos), (rate, kind, f0)


# ---- the state-variable form ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("rate", [8000, 16000, 48000])
def test_svf_params_reproduce_every_section(rate):
    from viettts_b200.engine import eq_sections
    filters = [eq_sections(s, rate) for s in ("telephone", VOICE if rate >= 16000 else "hp:80:4,pk:1000:1:3", "hp:60:8",
                                               "pk:100:30:12,ls:50:24,hs:3000:-24:0.3,notch:50:20,lp:10:1")]
    filters.append(elliptic_hp(rate))
    w = np.linspace(0, np.pi, 4097)[1:-1]
    for sos in filters:
        for row in sos:
            h = signal.sosfreqz(row[None], w)[1]
            hs = eo.svf_response(eo.svf_params(row[None]), w)
            assert np.abs(hs - h).max() <= 1e-11 * max(1.0, np.abs(h).max()), row


def test_svf_in_float64_equals_sosfilt():
    rate = 48000
    for sos in (eo.butter("highpass", 4, 60, rate), elliptic_hp(rate)):
        A, c = eo.transitions(sos)
        x = noise(4000, 1)
        s = np.zeros(2 * c.shape[0])
        y = np.array([eo._step64(c, s, v) for v in x])
        assert np.abs(y - eo.sosfilt(sos, x)).max() <= 1e-12


# ---- tolerance and the kernels' fp32 arithmetic ---------------------------------------------------------------------

def adversarial():
    """(name, sos, x) cases for the emulation"""
    cases = []
    r = 48000
    hp4 = eo.butter("highpass", 4, 60, r)
    cases.append(("50 Hz through HP4 60 Hz", hp4, tone(50, 3 * r // 2, r)))
    cases.append(("elliptic HP6", elliptic_hp(r), noise(r, 2)))
    cases.append(("Q=30 peak at 100 Hz", eo.peaking(100.0, 30.0, 24.0, r), tone(100, r, r)))
    cases.append(("+24 dB low shelf", eo.shelf(False, 100.0, 24.0, 1.0, r), noise(20000, 3)))
    cases.append(("+24 dB high shelf", eo.shelf(True, 4000.0, 24.0, 1.0, r), noise(20000, 4)))
    cases.append(("full-scale noise, worst", np.concatenate([eo.butter("highpass", 8, 60, r), eo.butter("lowpass", 8, 7000, r)]),
                  np.sign(noise(30000, 5))))
    cases.append(("clicks, telephone", np.concatenate([eo.butter("highpass", 4, 300, 8000), eo.butter("lowpass", 4, 3400, 8000)]),
                  clicks(9000)))
    return cases


def test_emulation_within_tolerance_on_adversarial_rows():
    for name, sos, x in adversarial():
        x = np.asarray(x, np.float32)
        e = error_units(eo.emulate(sos, x), eo.sosfilt(sos, x), x, sos)
        print(f"{name}: {e:.2f} units")
        assert e <= TOL / 4, name


def test_three_minute_row_emulation():
    rate = 16000
    from viettts_b200.engine import eq_sections
    sos = eq_sections(VOICE, rate)
    x = np.tile(noise(6 * rate, 6) * np.hanning(6 * rate), 30).astype(np.float32)
    e = error_units(eo.emulate(sos, x), eo.sosfilt(sos, x), x, sos)
    print(f"3 min: {e:.2f} units")
    assert e <= TOL / 4


def test_tolerance_has_headroom_over_the_emulation():
    worst = 0.0
    for _, sos, x in adversarial():
        x = np.asarray(x, np.float32)
        worst = max(worst, error_units(eo.emulate(sos, x), eo.sosfilt(sos, x), x, sos))
    print(f"fp32 emulation {worst:.2f} units (TOL {TOL})")
    assert 4 * worst <= TOL <= 16 * worst, worst


@pytest.mark.parametrize("pattern", ["one", "full", "random"])
def test_stream_emulation_gives_the_same_bits(pattern):
    sos = np.concatenate([eo.butter("highpass", 4, 80, 16000), eo.peaking(3000, 1.0, 3.0, 16000)])
    n = 1500 if pattern == "one" else 5000
    x = noise(n, 8).astype(np.float32)
    rng = np.random.default_rng(1)
    F = 700
    sizes, left = [], n
    while left:
        k = min(left, 1 if pattern == "one" else (F if pattern == "full" else int(rng.integers(0, F + 1))))
        sizes.append(k)
        left -= k
    got = np.concatenate(eo.emulate_stream(sos, x, sizes))
    assert np.array_equal(got, eo.emulate(sos, x))


# ---- spec parsing, validators and the CLI ---------------------------------------------------------------------------

def test_spec_parsing():
    from viettts_b200.engine import eq_sections
    lib()
    t = eq_sections("telephone", 8000)
    assert t.shape == (4, 6)
    assert np.array_equal(t, np.concatenate([eq_sections("hp:300:4", 8000), eq_sections("lp:3400:4", 8000)]))
    assert np.array_equal(eq_sections(" HP:80 , pk:3000:1:3", 16000),
                          np.concatenate([design(eo.HIGHPASS, 16000, 80.0, order=2)[1], design(eo.PEAKING, 16000, 3000.0, 1.0, 3.0)[1]]))
    assert np.array_equal(eq_sections("ls:200:-2", 16000), eq_sections("ls:200:-2:1", 16000))
    assert eq_sections(VOICE, 48000).shape == (5, 6)
    assert eq_sections(WORST, 48000).shape == (8, 6)
    e = elliptic_hp(48000)
    assert np.array_equal(eq_sections(e, 48000), e)


def test_sos_arrays_reach_the_library_row_major():
    """the library reads sos as C-order [K][6]: a Fortran-ordered or transposed input comes back as a row-major copy"""
    from viettts_b200.engine import eq_sections
    e = elliptic_hp(48000)
    for arr in (np.asfortranarray(e), np.ascontiguousarray(e.T).T, e[:, :], e[::-1][::-1], e.astype(np.float32)):
        got = eq_sections(arr, 48000)
        assert got.flags.c_contiguous and got.dtype == np.float64
        assert np.array_equal(got, np.asarray(e, np.float64) if arr.dtype == np.float64 else arr.astype(np.float64))
        assert np.array_equal(np.frombuffer(got.tobytes(order="A"), np.float64).reshape(-1, 6), got)


@pytest.mark.parametrize("spec,rate", [("hp:60:8,lp:7000:8,pk:100:1:1", 48000), ("telephone,telephone,hp:50", 8000), ("lp:3400", 7000),
                                       ("lp:3700", 8000), ("hp:5", 16000), ("pk:100:3", 16000), ("pk:100:0.05:3", 16000),
                                       ("ls:100:25", 16000), ("hs:100:3:2", 16000), ("hp:100:2.5", 16000), ("hp:abc", 16000),
                                       ("band:100", 16000), ("", 16000), ("notch:50", 16000), ("hp:100", 16000.5),
                                       ([[1, 0, 0, 1, -2.0, 1.0]], 16000), ([[1, 0, 0, 0, 0.1, 0.1]], 16000),
                                       ([[1, 0, 0, 1, float("nan"), 0.5]], 16000), (np.zeros((0, 6)), 16000),
                                       (np.tile([1.0, 0, 0, 1, 0, 0], (9, 1)), 16000), ([[1, 0, 0, 1, 0]], 16000),
                                       ([[1, 0, 0, 1, -1.9999999, 0.99999999]], 16000), ("hp:100", float("inf")),
                                       ("hp:100", float("nan")), ("hp:100", "fast"), ("hp:100:inf", 16000), ("hp:100:nan", 16000),
                                       ("pk:100:inf:3", 16000)])
def test_spec_rejections(spec, rate):
    from viettts_b200.engine import eq_sections
    lib()
    with pytest.raises(ValueError):
        eq_sections(spec, rate)


def test_validator_agrees_with_the_oracle():
    from viettts_b200.engine import _eq_stable
    rng = np.random.default_rng(3)
    for _ in range(2000):
        row = np.array([1.0, 0.3, -0.2, 1.0, *rng.uniform(-2.2, 2.2, 1), *rng.uniform(-1.2, 1.2, 1)])
        assert _eq_stable(row) == eo.valid(row[None]), row


@pytest.mark.parametrize("argv", [["--eq", "hp:5"], ["--eq", "telephone,telephone,hp:50"], ["--eq", "lp:3700", "--output-rate", "8000"],
                                  ["--eq", "wobble"], ["--eq", "pk:1000:1"], ["--eq", "hp:100:inf"], ["--eq", "hp:inf"]])
def test_cli_rejects_bad_eq(argv):
    from viettts_b200 import synthesizer
    lib()
    with pytest.raises(SystemExit):
        synthesizer.main(["--text", "xin chào", *argv])
