"""GPU: the equalizer (Engine.equalize / equalize_forward, vtts_eq*), its stream (Engine.open_eq_stream), the TTS stream's
`eq=` stage and the CLI's --eq.

One-shot outputs are held to the float64 definition (scipy.signal.sosfilt) within TOL error units
(tests/test_eq_cpu.py, over 4x an fp32 emulation of the kernels); everything that streams, and every precision mode and
batch position, is compared bit for bit with the one-shot call."""
import ctypes
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import eq_oracle as eo
from test_eq_cpu import TOL, VOICE, WORST, clicks, elliptic_hp, error_units, noise, tone
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def rows(rate, lengths, seed=0):
    S = max(lengths)
    x = np.zeros((len(lengths), S), np.float32)
    kinds = [lambda n: tone(50, n, rate), lambda n: clicks(n) if n >= 8 else noise(n, seed), lambda n: noise(n, seed),
             lambda n: np.sign(noise(n, seed + 1))]
    for b, n in enumerate(lengths):
        if n:
            x[b, :n] = kinds[b % 4](n)
    return x


def filters(rate):
    """the four filters where their bands fit the rate"""
    out = [("telephone", "telephone")]
    if rate >= 16000:
        out.append(("voice", VOICE))
        out.append(("worst", WORST))
    out.append(("elliptic", elliptic_hp(rate)))
    return out


@pytest.mark.parametrize("rate", [8000, 16000, 44100, 48000])
def test_ragged_rows_against_float64(eng, rate):
    from viettts_b200.engine import eq_sections
    lengths = [rate // 3, 1, 0, 3 * 1024 + 777, rate // 2, 1024, 45]
    x = rows(rate, lengths, rate)
    for name, spec in filters(rate):
        sos = eq_sections(spec, rate)
        y = eng.equalize(x, spec, rate, lengths=lengths)
        for b, n in enumerate(lengths):
            assert np.all(y[b, n:] == 0), (name, b)
            if n:
                e = error_units(y[b, :n], eo.sosfilt(sos, x[b, :n]), x[b, :n], sos)
                assert e <= TOL, (name, b, e)


def test_three_minute_row(eng):
    from viettts_b200.engine import eq_sections
    rate = 16000
    sos = eq_sections(VOICE, rate)
    x = np.tile(noise(6 * rate, 6) * np.hanning(6 * rate), 30).astype(np.float32)
    y = eng.equalize(x, VOICE, rate)
    assert error_units(y, eo.sosfilt(sos, x), x, sos) <= TOL


def test_same_bits_in_every_mode_and_batch_position(eng):
    rate = 48000
    x = rows(rate, [5000, 3000, 7000, 6000], 9)
    base = eng.equalize(x, WORST, rate)
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            assert np.array_equal(eng.equalize(x, WORST, rate), base), mode
    finally:
        eng.set_precision("bf16x3")
    for b in range(4):
        assert np.array_equal(eng.equalize(x[b], WORST, rate), base[b]), b
        perm = np.roll(np.arange(4), b)
        assert np.array_equal(eng.equalize(x[perm], WORST, rate), base[perm]), b


def test_forward_in_place_and_device_lengths(eng):
    rate = 48000
    x = rows(rate, [20000, 9000], 2)
    ref = eng.equalize(x, VOICE, rate, lengths=[20000, 9000])
    x_t = torch.from_numpy(x).cuda()
    n_t = torch.tensor([20000, 9000], dtype=torch.int32, device="cuda")
    y_t = eng.equalize_forward(x_t.clone(), VOICE, rate, lengths_t=n_t)
    assert np.array_equal(y_t.cpu().numpy(), ref)
    y_t = eng.equalize_forward(x_t, VOICE, rate, lengths_t=n_t, out=x_t)
    assert y_t.data_ptr() == x_t.data_ptr()
    assert np.array_equal(y_t.cpu().numpy(), ref)


def test_fortran_ordered_sos_runs_the_same_filter(eng):
    rate = 48000
    e = elliptic_hp(rate)
    x = rows(rate, [9000, 4000], 3)
    ref = eng.equalize(x, e, rate)
    for arr in (np.asfortranarray(e), np.ascontiguousarray(e.T).T):
        assert not arr.flags.c_contiguous
        assert np.array_equal(eng.equalize(x, arr, rate), ref)
        x_t = torch.from_numpy(x).cuda()
        assert np.array_equal(eng.equalize_forward(x_t, arr, rate).cpu().numpy(), ref)
        with eng.open_eq_stream(2, 9000, arr, rate) as st:
            ys = st.push(x, [9000, 4000], [True, True], [True, True])
        assert np.array_equal(ys[0], ref[0]) and np.array_equal(ys[1], ref[1, :4000])


@pytest.mark.parametrize("S", [1, 3, 32])
@pytest.mark.parametrize("pattern", ["one", "full", "random"])
def test_stream_equals_one_shot(eng, S, pattern):
    """rows pushed in `pattern` chunks (through push_device, in place, for "random") and held to the stream's
    contract on every push (tests/helpers/slot_streams.py)"""
    rate = 16000
    lengths = [int(v) for v in np.random.default_rng(S).integers(1, 2500 if pattern == "one" else 9000, size=S)]
    x = rows(rate, lengths, S)
    rng = np.random.default_rng(7)
    stage = ss.stage(eng, "eq", S, 700, rate, eq=VOICE)
    ss.run(stage, [[ss.pattern(pattern, n, 700, rng)] for n in lengths], lambda s, u, n: x[s, :n], host=pattern != "random")


def test_launch_counts(eng):
    rate = 16000
    x = rows(rate, [4000], 1)
    with eng.open_eq_stream(1, 500, WORST, rate) as st:
        for i in range(8):
            c0 = eng.launch_count()
            ys = st.push(x[:, 500 * i:500 * i + 500], [500], [i == 0], [i == 7])
            assert eng.launch_count() - c0 == 4
            assert ys[0].size == 500
    for spec in ("hp:100:1", WORST):
        c0 = eng.launch_count()
        eng.equalize(np.zeros((3, 50000), np.float32), spec, rate)
        assert eng.launch_count() - c0 == 3


def test_argument_errors(eng):
    from viettts_b200 import _lib
    x = np.zeros((2, 100), np.float32)
    unstable = [[1.0, 0, 0, 1.0, -2.0, 1.0]]
    for spec in (unstable, np.zeros((0, 6)), np.tile([1.0, 0, 0, 1, 0, 0], (9, 1)), "hp:7300", "pk:100:1:nan",
                 [[1.0, 0, 0, 1.0, float("nan"), 0.5]]):
        with pytest.raises(ValueError):
            eng.equalize(x, spec, 16000)
    with pytest.raises(ValueError):
        eng.equalize(x, "hp:100", 16000, lengths=[1, 2, 3])
    lib = eng.lib
    y = np.zeros_like(x)
    for sos, K in ((np.array(unstable), 1), (np.tile([1.0, 0, 0, 1, 0, 0], (9, 1)), 0), (np.tile([1.0, 0, 0, 1, 0, 0], (9, 1)), 9),
                   (np.array([[1.0, 0, 0, 1.0, float("nan"), 0.5]]), 1)):
        with pytest.raises(_lib.VttsError, match="K=|section"):
            eng._ck(lib.vtts_eq_host(eng.h, x.ctypes.data, None, 2, 100, sos.ctypes.data, K, y.ctypes.data))
    good = np.array([[1.0, 0, 0, 1, 0, 0]])
    n = np.array([5, 200], np.int32)
    with pytest.raises(_lib.VttsError, match="outside"):
        eng._ck(lib.vtts_eq_host(eng.h, x.ctypes.data, n.ctypes.data, 2, 100, good.ctypes.data, 1, y.ctypes.data))
    with pytest.raises(_lib.VttsError):
        eng._ck(lib.vtts_eq_host(eng.h, x.ctypes.data, None, 0, 100, good.ctypes.data, 1, y.ctypes.data))
    with pytest.raises(_lib.VttsError, match="section 0"):
        h = ctypes.c_void_p()
        eng._ck(lib.vtts_eq_stream_create(eng.h, 2, 64, np.array(unstable).ctypes.data, 1, ctypes.byref(h)))
    with eng.open_eq_stream(2, 64, "hp:100") as st:
        with pytest.raises(_lib.VttsError, match="not open"):
            st.push(np.zeros((2, 64), np.float32), [64, 0], None, None)
        with pytest.raises(_lib.VttsError, match="outside"):
            st.push(np.zeros((2, 64), np.float32), [65, 0], [True, False], None)
        with pytest.raises(ValueError):
            st.push(np.zeros((2, 65), np.float32), [64, 0], [True, False], None)


@pytest.fixture(scope="module")
def tts_eng(acoustic_ckpt, hifigan_params):
    from viettts_b200.engine import Engine
    e = Engine(0)
    e.load_acoustic(acoustic_ckpt)
    e.load_hifigan(hifigan_params)
    e.load_duration(synthetic.duration_ckpt(1234))
    yield e
    e.close()


def tts_tokens(seed, L):
    rng = np.random.default_rng(seed)
    t = rng.integers(4, 90, size=L).astype(np.int32)
    t[4::5] = 3
    t[0] = t[-1] = 0
    return t


def test_tts_stream_eq(tts_eng):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(150 + b, n) for b, n in enumerate([25, 40])]
        audio = {0: [], 1: []}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=8000, eq="telephone", limit=-3.0) as ts:
            assert ts.eq is not None and ts.eq.lookahead == 0
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
        for s in (0, 1):
            w = eng.tts(toks[s][None], silence_duration=0.1)[0][0]
            w = eng.limit(eng.equalize(eng.resample(w, 8000), "telephone", 8000), -3.0, 8000)[0]
            assert np.array_equal(np.concatenate(audio[s]), w), s
        with pytest.raises(ValueError):
            eng.open_tts_stream(1, 16, 2000, 100, eq="lp:7500")
    finally:
        eng.set_fused_pairs(True)


def test_cli_eq(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
    from viettts_b200 import synthesizer
    from viettts_b200.engine import get_engine
    from viettts_b200.hifigan.mel2wave import mel2wave
    from viettts_b200.nat.text2mel import text2mel
    (tmp_path / "assets/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/hifigan").mkdir(parents=True)
    (tmp_path / "assets/infore/nat").mkdir(parents=True)
    (tmp_path / "assets/hifigan/config.json").write_text(json.dumps(config.HIFIGAN))
    for path, obj in (("assets/infore/hifigan/hk_hifi.pickle", hifigan_params), ("assets/infore/nat/acoustic_latest_ckpt.pickle", acoustic_ckpt),
                      ("assets/infore/nat/duration_latest_ckpt.pickle", synthetic.duration_ckpt(1234))):
        with open(tmp_path / path, "wb") as f:
            pickle.dump(obj, f)
    monkeypatch.chdir(tmp_path)
    lex = str(golden_dir / "lexicon_small.txt")
    ge = get_engine(0)
    text = "Xin chào, tôi là trợ lý ảo."
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    assert synthesizer.main(["--text", text, "--output", "one.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--eq", "telephone", "--output-rate", "8000"]) == 0
    expect = synthesizer.float_to_pcm16(ge.equalize(ge.resample(wave, 8000), "telephone", 8000)).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
