"""GPU: the split-band de-esser (Engine.deess / deess_forward, vtts_deess*), its stream (Engine.open_deesser_stream), the
TTS stream's `deess=` stage and the CLI's --deess.

One-shot outputs are held to the float64 definition (oracle/deesser_oracle.py) within TOL error units
(tests/test_deesser_cpu.py, over 4x an fp32 emulation of the kernels); everything that streams, and every precision
mode and batch position, is compared bit for bit with the one-shot call."""
import ctypes
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import deesser_oracle as do
from test_deesser_cpu import PARAMS, TOL, cases, clear_of_bursts, error_units, parts, sibilant_speech
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def rows(rate, lengths, seed=0):
    S = max(max(lengths), 1)
    x = np.zeros((len(lengths), S), np.float32)
    for b, n in enumerate(lengths):
        if n:
            x[b, :n] = cases(rate, n)[(b + seed) % 6]
    return x


def check_rows(y, red, x, lengths, rate, kw, what):
    for b, n in enumerate(lengths):
        assert np.all(y[b, n:] == 0), (what, b)
        if n == 0:
            assert red[b] == 0, (what, b)
            continue
        ref, rref, P = parts(x[b, :n], rate, **kw)
        e = error_units(y[b, :n], ref, x[b, :n], P)
        assert e <= TOL, (what, b, n, e)
        assert abs(float(red[b]) - rref) <= 1e-3 * max(1.0, abs(rref)), (what, b, red[b], rref)


@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_ragged_rows_against_float64(eng, rate):
    lengths = [0, 1, 255, 256, 257, 1023, 1024, 1025, rate // 2, rate]
    for name, kw in PARAMS.items():
        x = rows(rate, lengths, len(name))
        y, red = eng.deess(x, kw, rate, lengths=lengths)
        check_rows(y, red, x, lengths, rate, kw, name)


def test_three_minute_row(eng):
    rate = 16000
    x = np.tile(sibilant_speech(6 * rate, rate, 4, -6.0)[0], 30)
    y, red = eng.deess(x, "voice", rate)
    ref, rref, P = parts(x, rate)
    assert error_units(y, ref, x, P) <= TOL
    assert rref < 0 and abs(float(red) - rref) <= 1e-3 * abs(rref)


def test_pass_through_is_bit_exact(eng):
    rate = 16000
    quiet = (0.05 * np.sin(2 * np.pi * 300 / rate * np.arange(20000))).astype(np.float32)      # no high band above the knee
    loud, _ = sibilant_speech(20000, rate, 2, -3.0)
    for x, kw in ((quiet, {}), (quiet, dict(freq=2000.0)), (loud, dict(ratio=1.0)), (loud, dict(range=0.0))):
        y, red = eng.deess(x, kw, rate)
        assert red == 0.0 and np.array_equal(y, x), kw
    x = np.stack([quiet, np.zeros_like(quiet)])
    y, red = eng.deess(x, "voice", rate, lengths=[12345, 0])
    assert np.array_equal(y[0, :12345], quiet[:12345]) and np.all(y[0, 12345:] == 0) and np.all(y[1] == 0)


@pytest.mark.parametrize("rate", [16000, 48000])
def test_bursts_are_turned_down_and_the_rest_is_not(eng, rate):
    x, mask = sibilant_speech(rate, rate, 4, -6.0)
    y, red = eng.deess(x, "release=5", rate)
    _, _, P = parts(x, rate, release=5.0)
    off = clear_of_bursts(mask, rate)
    assert off.sum() > 0.1 * rate and np.array_equal(y[off], x[off])
    high = y.astype(np.float64) - (x.astype(np.float64) - P["h"])        # the split's high band of y: g h
    assert np.sum(high[mask] ** 2) < 10 ** (-6 / 10) * np.sum(P["h"][mask] ** 2)
    assert -12.0 <= red < -6.0


def test_same_bits_in_every_mode_and_batch_position(eng):
    rate = 48000
    x = rows(rate, [5000, 3000, 7000, 6000], 1)
    base, rb = eng.deess(x, "voice", rate)
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            y, r = eng.deess(x, "voice", rate)
            assert np.array_equal(y, base) and np.array_equal(r, rb), mode
    finally:
        eng.set_precision("bf16x3")
    for b in range(4):
        y1, r1 = eng.deess(x[b], "voice", rate)
        assert np.array_equal(y1, base[b]) and r1 == rb[b], b
        perm = np.roll(np.arange(4), b)
        yp, rp = eng.deess(x[perm], "voice", rate)
        assert np.array_equal(yp, base[perm]) and np.array_equal(rp, rb[perm]), b


def test_forward_in_place_and_device_reduction(eng):
    rate = 48000
    x = rows(rate, [20000, 9000], 2)
    ref, rr = eng.deess(x, "ratio=6", rate, lengths=[20000, 9000])
    assert rr.min() < 0
    x_t = torch.from_numpy(x).cuda()
    n_t = torch.tensor([20000, 9000], dtype=torch.int32, device="cuda")
    y_t, r_t = eng.deess_forward(x_t, "ratio=6", rate, lengths_t=n_t, out=x_t)
    assert y_t.data_ptr() == x_t.data_ptr() and r_t.is_cuda
    assert np.array_equal(y_t.cpu().numpy(), ref) and np.array_equal(r_t.cpu().numpy(), rr)


@pytest.mark.parametrize("S", [1, 3, 32])
@pytest.mark.parametrize("pattern,device", [("one", False), ("full", False), ("full", True), ("random", False), ("random", True)])
def test_stream_equals_one_shot(eng, S, pattern, device):
    """rows pushed in `pattern` chunks (device pushes in place) and held to the stream's contract on every push
    (tests/helpers/slot_streams.py)"""
    rate = 48000
    if pattern == "one" and S == 32:
        pytest.skip("one-sample pushes run at S = 1 and 3")
    # lengths and chunks across both block sizes (256 and 1024)
    lengths = [int(v) for v in np.random.default_rng(S).integers(1, 2500 if pattern == "one" else 12000, size=S)]
    x = rows(rate, lengths, S)
    rng = np.random.default_rng(7)
    for chunk in (700, 1500):
        stage = ss.stage(eng, "deesser", S, chunk, rate, spec="attack=0.5,release=20,threshold=-40")
        out = ss.run(stage, [[ss.pattern(pattern, n, chunk, rng)] for n in lengths], lambda s, u, n: x[s, :n], host=not device)
        assert min(row[0][3] for row in out) < 0
        if pattern == "one":
            break


def test_launch_counts(eng):
    rate = 16000
    x = rows(rate, [4000], 0)
    with eng.open_deesser_stream(1, 500, "voice", rate) as st:
        for i in range(8):
            c0 = eng.launch_count()
            ys = st.push(x[:, 500 * i:500 * i + 500], [500], [i == 0], [i == 7])
            assert eng.launch_count() - c0 == 10
            assert ys[0].size == 500
    with eng.open_deesser_stream(32, 3000, "voice", rate) as st:
        c0 = eng.launch_count()
        st.push(np.zeros((32, 3000), np.float32), np.full(32, 3000), np.ones(32, bool), None)
        assert eng.launch_count() - c0 == 10
    for shape in ((3, 50000), (1, 10)):
        c0 = eng.launch_count()
        eng.deess(np.zeros(shape, np.float32), "voice", rate)
        assert eng.launch_count() - c0 == 9


def test_argument_errors(eng):
    from viettts_b200 import _lib
    x = np.zeros((2, 100), np.float32)
    for spec in ("freq=900", "freq=7300", "ratio=0.5", "threshold=1", "knee=-1", "attack=0.4", "release=4", "range=25",
                 "range=nan", "makeup=1"):
        with pytest.raises(ValueError):
            eng.deess(x, spec)
    with pytest.raises(ValueError, match="freq"):
        eng.deess(x, "voice", 8000)
    with pytest.raises(ValueError):
        eng.deess(x, "voice", lengths=[1, 2, 3])
    lib = eng.lib
    y = np.zeros_like(x)
    good = (5000.0, -30.0, 4.0, 6.0, 1.0, 60.0, 12.0)
    c0 = eng.launch_count()
    for i, bad in ((0, float("nan")), (0, 999.0), (0, 7201.0), (1, float("nan")), (1, -61.0), (2, 0.9), (2, 21.0), (3, -0.1),
                   (3, 25.0), (4, 0.4), (4, 201.0), (5, 4.9), (5, 5001.0), (6, -0.1), (6, 24.5), (6, float("nan"))):
        p = list(good)
        p[i] = bad
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_deess_host(eng.h, x.ctypes.data, None, 2, 100, 16000, *p, y.ctypes.data, None))
    with pytest.raises(_lib.VttsError, match="freq"):
        eng._ck(lib.vtts_deess_host(eng.h, x.ctypes.data, None, 2, 100, 8000, *good, y.ctypes.data, None))
    for B, S, rate in ((0, 100, 16000), (2, 0, 16000), (2, 100, 7999), (2, 100, 192001)):
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_deess_host(eng.h, x.ctypes.data, None, B, S, rate, *good, y.ctypes.data, None))
    n = np.array([5, 200], np.int32)
    with pytest.raises(_lib.VttsError, match="outside"):
        eng._ck(lib.vtts_deess_host(eng.h, x.ctypes.data, n.ctypes.data, 2, 100, 16000, *good, y.ctypes.data, None))
    h = ctypes.c_void_p()
    with pytest.raises(_lib.VttsError, match="range"):
        eng._ck(lib.vtts_deesser_stream_create(eng.h, 2, 64, 16000, 5000.0, -30.0, 4.0, 6.0, 1.0, 60.0, 30.0, ctypes.byref(h)))
    with pytest.raises(_lib.VttsError, match="freq"):
        eng._ck(lib.vtts_deesser_stream_create(eng.h, 2, 64, 8000, *good, ctypes.byref(h)))
    with pytest.raises(_lib.VttsError, match="max_streams"):
        eng._ck(lib.vtts_deesser_stream_create(eng.h, 0, 64, 16000, *good, ctypes.byref(h)))
    assert eng.launch_count() == c0
    with eng.open_deesser_stream(2, 64) as st:
        with pytest.raises(_lib.VttsError, match="not open"):
            st.push(np.zeros((2, 64), np.float32), [64, 0], None, None)
        with pytest.raises(_lib.VttsError, match="outside"):
            st.push(np.zeros((2, 64), np.float32), [65, 0], [True, False], None)
        with pytest.raises(ValueError):
            st.push(np.zeros((2, 65), np.float32), [64, 0], [True, False], None)
        with pytest.raises(ValueError, match="reduction_t"):
            st.push_device(torch.zeros((2, 64), device="cuda"), [64, 0], np.array([1, 0], np.uint8), torch.zeros((2, 64), device="cuda"),
                           torch.zeros(3, device="cuda"))
    assert eng.launch_count() == c0


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


@pytest.mark.parametrize("rate,compress,limit", [(None, None, None), (None, "threshold=-30,ratio=4", -1.0), (48000, None, None),
                                                 (48000, "voice", -3.0)])
def test_tts_stream_deess(tts_eng, rate, compress, limit):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(160 + b, n) for b, n in enumerate([25, 40])]
        audio = {0: [], 1: []}
        spec = "threshold=-50,ratio=4"
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, compress=compress, deess=spec, limit=limit) as ts:
            assert ts.ds is not None and ts.ds.lookahead == 0
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
        chain = AudioChain(output_rate=rate, compress=compress, deess=spec, limit=limit)
        for s in (0, 1):
            w = chain.run(eng, eng.tts(toks[s][None], silence_duration=0.1)[0][0])
            assert np.array_equal(np.concatenate(audio[s]), w), s
        with pytest.raises(ValueError, match="deess"):
            eng.open_tts_stream(1, 16, 2000, 100, deess="range=30")
    finally:
        eng.set_fused_pairs(True)


def test_cli_deess(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
                             "--deess", "voice", "--output-rate", "48000"]) == 0
    expect = synthesizer.float_to_pcm16(ge.deess(ge.resample(wave, 48000), "voice", 48000)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
    assert synthesizer.main(["--text", text, "--output", "two.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--compress", "threshold=-30,ratio=4", "--deess", "threshold=-50,range=6", "--loudness", "-16",
                             "--limiter"]) == 0
    c = ge.compress(wave, "threshold=-30,ratio=4", 16000)[0]
    d = ge.deess(c, "threshold=-50,range=6", 16000)[0]
    expect = synthesizer.float_to_pcm16(ge.normalize_loudness(d, -16.0, 16000, true_peak=-1.0, limit=True)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "two.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
