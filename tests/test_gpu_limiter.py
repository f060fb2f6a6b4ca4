"""GPU: the lookahead true-peak limiter (Engine.limit / limit_forward, vtts_limit*), its stream
(Engine.open_limiter_stream), loudness normalization through it (normalize_loudness(limit=True)), the TTS stream's
`limit=` stage and the CLI's --limiter.

One-shot outputs are held to the float64 definition within Y_TOL error units (tests/test_limiter_cpu.py, over 4x an
fp32 emulation of the kernels); everything that streams, and every precision mode and batch position, is compared bit
for bit with the one-shot call."""
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import limiter_oracle as lm
from oracle import loudness_oracle as lo
from test_limiter_cpu import TP_MARGIN, Y_TOL, clicks, error_units, fs4_sine, noise, speech_like
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
    kinds = [lambda n: fs4_sine(n), lambda n: clicks(n) if n >= 8 else noise(n, seed), lambda n: noise(n, seed), lambda n: speech_like(n / rate + 0.01, rate, seed)[:n]]
    for b, n in enumerate(lengths):
        if n:
            x[b, :n] = kinds[b % 4](n)
    return x


@pytest.mark.parametrize("rate", [8000, 16000, 44100, 48000])
def test_ragged_rows_against_float64(eng, rate):
    lengths = [rate // 3, 1, 0, 777, rate // 2, 45]
    x = rows(rate, lengths, rate)
    gains = np.array([0.0, 6.0, -3.0, 20.0, 12.0, 40.0], np.float32)
    y, red = eng.limit(x, -1.0, rate, gain_db=gains, lookahead_ms=3.0, release_ms=60.0, lengths=lengths)
    c = 10 ** (-1.0 / 20)
    for b, n in enumerate(lengths):
        assert np.all(y[b, n:] == 0), b
        if n == 0:
            assert red[b] == 0
            continue
        ref, rref, P = lm.limit(x[b, :n], rate, -1.0, gains[b], 3.0, 60.0, parts=True)
        assert error_units(y[b, :n], ref, P) <= Y_TOL, (b, error_units(y[b, :n], ref, P))
        assert np.abs(y[b, :n]).max() <= np.float32(c) * (1 + 2 ** -22)
        assert abs(float(red[b]) - rref) <= 1e-3 or (np.isinf(rref) and np.isinf(red[b])), (b, red[b], rref)


def test_three_minute_row(eng):
    rate = 16000
    x = np.tile(speech_like(6.0, rate, 4), 30)
    y, red = eng.limit(x, -2.0, rate, gain_db=8.0)
    ref, rref, P = lm.limit(x, rate, -2.0, 8.0, parts=True)
    assert error_units(y, ref, P) <= Y_TOL
    assert abs(float(red) - rref) <= 1e-3


@pytest.mark.parametrize("rate", [16000, 48000])
def test_output_true_peak_under_the_ceiling(eng, rate):
    n = rate // 4
    x = np.stack([fs4_sine(n), clicks(n), noise(n, 1, 1.0), speech_like(n / rate, rate, 3)[:n]]).astype(np.float32)
    y, _ = eng.limit(x, -1.0, rate, gain_db=20.0)
    for b in range(4):
        assert lo.true_peak(y[b]) <= -1.0 + TP_MARGIN, b


def test_pass_through_is_bit_exact(eng):
    x = (0.2 * np.sin(2 * np.pi * 300 / 16000 * np.arange(16000))).astype(np.float32)
    for g in (0.0, 3.0, -10.0):
        y, red = eng.limit(x, -1.0, 16000, gain_db=g)
        assert red == 0.0
        assert np.array_equal(y, lm.gain_factor(g) * x), g


def test_same_bits_in_every_mode_and_batch_position(eng):
    rate = 16000
    x = rows(rate, [5000, 3000, 7000, 6000], 9)
    base, rb = eng.limit(x, -3.0, rate, gain_db=10.0)
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            y, r = eng.limit(x, -3.0, rate, gain_db=10.0)
            assert np.array_equal(y, base) and np.array_equal(r, rb), mode
    finally:
        eng.set_precision("bf16x3")
    for b in range(4):
        y1, r1 = eng.limit(x[b], -3.0, rate, gain_db=10.0)
        assert np.array_equal(y1, base[b]) and r1 == rb[b], b
        perm = np.roll(np.arange(4), b)
        yp, rp = eng.limit(x[perm], -3.0, rate, gain_db=10.0)
        assert np.array_equal(yp, base[perm]) and np.array_equal(rp, rb[perm]), b


def test_forward_in_place_and_device_gain(eng):
    rate = 48000
    x = rows(rate, [20000, 9000], 2)
    g = np.array([6.0, 15.0], np.float32)
    ref, rr = eng.limit(x, -1.0, rate, gain_db=g, lengths=[20000, 9000])
    x_t = torch.from_numpy(x).cuda()
    n_t = torch.tensor([20000, 9000], dtype=torch.int32, device="cuda")
    y_t, r_t = eng.limit_forward(x_t, -1.0, rate, gain_db=torch.from_numpy(g).cuda(), lengths_t=n_t, out=x_t)
    assert y_t.data_ptr() == x_t.data_ptr()
    assert np.array_equal(y_t.cpu().numpy(), ref) and np.array_equal(r_t.cpu().numpy(), rr)


@pytest.mark.parametrize("S", [1, 3, 32])
@pytest.mark.parametrize("pattern", ["one", "full", "random"])
def test_stream_equals_one_shot(eng, S, pattern):
    """rows pushed in `pattern` chunks through the host push, each slot at its own pre-gain, and held to the stream's
    contract on every push (tests/helpers/slot_streams.py)"""
    rate = 16000
    if pattern == "one" and S == 32:
        pytest.skip("one-sample pushes run at S = 1 and 3")
    lengths = [int(v) for v in np.random.default_rng(S).integers(1, 2500 if pattern == "one" else 9000, size=S)]
    x = rows(rate, lengths, S)
    gains = np.linspace(-6, 24, S).astype(np.float32)
    rng = np.random.default_rng(7)
    stage = ss.stage(eng, "limiter", S, 700, rate, ceiling=-1.0, lookahead_ms=3.0, release_ms=60.0)
    ss.run(stage, [[ss.pattern(pattern, n, 700, rng)] for n in lengths], lambda s, u, n: x[s, :n],
           [[float(g)] for g in gains], host=True)


def test_stream_schedule_and_launch_counts(eng):
    rate = 16000
    look = eng.limiter_stream_lookahead(rate, 3.0)
    assert look == lm.stream_lookahead(lm.params(rate, 3.0, 60.0)[0])
    x = rows(rate, [4000], 1)
    with eng.open_limiter_stream(1, 500, rate, -1.0, 3.0, 60.0) as st:
        P, E = 0, 0
        for i in range(8):
            c0 = eng.launch_count()
            ys = st.push(x[:, P:P + 500], [500], [i == 0], [i == 7], gain_db=6.0)
            assert eng.launch_count() - c0 == 9
            P += 500
            want = P if i == 7 else max(0, P - look)
            assert ys[0].size == want - E
            E = want
    c0 = eng.launch_count()
    eng.limit(x, -1.0, rate)
    assert eng.launch_count() - c0 == 8


def test_argument_errors(eng):
    x = np.zeros((2, 100), np.float32)
    for kw in (dict(ceiling=0.5), dict(ceiling=-21), dict(rate=16001), dict(lookahead_ms=0.5), dict(lookahead_ms=25),
               dict(release_ms=0.2), dict(gain_db=71), dict(gain_db=[1, 2, 3]), dict(gain_db=float("nan"))):
        with pytest.raises(ValueError):
            eng.limit(x, **kw)
    with pytest.raises(ValueError):
        eng.limit(x, lengths=[1, 2, 3])
    from viettts_b200 import _lib
    lib = eng.lib
    y = np.zeros_like(x)
    with pytest.raises(_lib.VttsError):
        eng._ck(lib.vtts_limit_host(eng.h, x.ctypes.data, None, None, 2, 100, 16000, 1.0, 5.0, 100.0, y.ctypes.data, None))
    n = np.array([5, 200], np.int32)
    with pytest.raises(_lib.VttsError, match="outside"):
        eng._ck(lib.vtts_limit_host(eng.h, x.ctypes.data, n.ctypes.data, None, 2, 100, 16000, -1.0, 5.0, 100.0, y.ctypes.data, None))
    with eng.open_limiter_stream(2, 64) as st:
        with pytest.raises(ValueError):
            st.push(np.zeros((2, 64), np.float32), [64, 0], [True, True], None, gain_db=[0.0, 99.0])
        with pytest.raises(_lib.VttsError, match="not open"):
            st.push(np.zeros((2, 64), np.float32), [64, 0], None, None)


def test_normalize_limited(eng):
    rate = 16000
    x = speech_like(6.0, rate, 1)
    y, g = eng.normalize_loudness(x, -16.0, rate, true_peak=-1.0, limit=True)
    yc, gc = eng.normalize_loudness(x, -16.0, rate, true_peak=-1.0)
    yref, gref = lm.normalize_limited(x, rate, -16.0, -1.0)
    assert abs(float(g) - gref) <= 2e-3, (g, gref)
    ref, _, P = lm.limit(x, rate, -1.0, float(g), parts=True)
    assert error_units(y, ref, P) <= Y_TOL
    Ly, Lc = lo.measure(y, rate)[0], lo.measure(yc, rate)[0]
    assert Ly > Lc + 2.0 and abs(Ly + 16.0) < 1.5, (Ly, Lc)
    assert lo.true_peak(y) <= -1.0 + TP_MARGIN
    # the default keeps today's capped gain; the forward form runs in place with the same bits
    x2 = np.stack([x, 0.1 * x, np.zeros_like(x)])
    yh, gh = eng.normalize_loudness(x2, -16.0, rate, true_peak=-1.0, limit=True)
    assert np.array_equal(yh[0], y) and gh[2] == 0 and np.array_equal(yh[2], x2[2])
    x_t = torch.from_numpy(x2).cuda()
    c0 = eng.launch_count()
    y_t, g_t = eng.normalize_loudness_forward(x_t, -16.0, rate, true_peak=-1.0, limit=True, out=x_t)
    torch.cuda.synchronize()
    assert eng.launch_count() - c0 == 30
    assert np.array_equal(y_t.cpu().numpy(), yh) and np.array_equal(g_t.cpu().numpy(), gh)
    with pytest.raises(ValueError):
        eng.normalize_loudness(x, -16.0, rate, limit=True)


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


@pytest.mark.parametrize("rate", [None, 48000])
def test_tts_stream_limit(tts_eng, rate):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(130 + b, n) for b, n in enumerate([25, 40])]
        sr = rate or config.SAMPLE_RATE
        audio = {0: [], 1: []}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, limit=-6.0, gain_db=12.0) as ts:
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1, gain_db=20.0)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
        for s, g in ((0, 12.0), (1, 20.0)):
            w = eng.tts(toks[s][None], silence_duration=0.1)[0][0]
            if rate:
                w = eng.resample(w, rate)
            a = np.concatenate(audio[s])
            assert np.array_equal(a, eng.limit(w, -6.0, sr, gain_db=g)[0]), s
        with eng.open_tts_stream(1, 16, 2000, 100) as ts:
            with pytest.raises(ValueError, match="limit"):
                ts.begin(0, toks[0], gain_db=3.0)
    finally:
        eng.set_fused_pairs(True)


def test_cli_limiter(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
                             "--limiter", "--true-peak", "-3", "--output-rate", "48000"]) == 0
    expect = synthesizer.float_to_pcm16(ge.limit(ge.resample(wave, 48000), -3.0, 48000)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
    assert synthesizer.main(["--text", text, "--output", "two.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--loudness", "-16", "--limiter"]) == 0
    expect = synthesizer.float_to_pcm16(ge.normalize_loudness(wave, -16.0, 16000, true_peak=-1.0, limit=True)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "two.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
