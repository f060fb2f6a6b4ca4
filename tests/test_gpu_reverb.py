"""GPU: the convolution reverb (Engine.reverb / reverb_forward, vtts_reverb*), its stream (Engine.open_reverb_stream), the
TTS stream's `reverb=` stage and the CLI's --reverb.

One-shot outputs are held to the float64 definition (oracle/reverb_oracle.py) within TOL error units
(tests/test_reverb_cpu.py, over 4x an fp32 emulation of the kernels); everything that streams, and every precision
mode and batch position, is compared bit for bit with the one-shot call."""
import ctypes
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import reverb_oracle as ro
from test_reverb_cpu import TOL, cases, error_units
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


def user_ir(L, rate, seed=0):
    rng = np.random.default_rng(L + seed)
    return (rng.standard_normal(L) * np.exp(-np.arange(L) / (0.3 * rate)) * 0.1).astype(np.float32)


def specs(rate):
    out = {"room": "room", "hall": "hall"}
    for L in (1, 511, 512, 513, 5 * rate):
        out[f"ir{L}"] = {"ir": user_ir(L, rate), "mix": 0.6}
    return out


def check_rows(y, x, lengths, rate, spec, what):
    from viettts_b200.engine import reverb_params
    p = reverb_params(spec, rate)
    for b, n in enumerate(lengths):
        assert np.all(y[b, n:] == 0), (what, b)
        if n == 0:
            continue
        ref = ro.reverb(x[b, :n], p["ir"], p["mix"])
        e = error_units(y[b, :n], ref, x[b, :n], p["ir"], p["mix"])
        assert e <= TOL, (what, b, n, e)


@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_ragged_rows_against_float64(eng, rate):
    lengths = [0, 1, 511, 512, 513, 1023, 1024, 1025, rate // 2, rate]
    for name, spec in specs(rate).items():
        x = rows(rate, lengths, len(name))
        y = eng.reverb(x, spec, rate, lengths=lengths)
        check_rows(y, x, lengths, rate, spec, name)


def test_three_minute_row(eng):
    rate = 16000
    x = np.tile(cases(rate, 6 * rate)[4], 30)
    y = eng.reverb(x, "hall", rate)
    check_rows(y[None], x[None], [x.size], rate, "hall", "3 min")


def test_mix_zero_is_bit_exact_and_an_impulse_delays(eng):
    rate = 48000
    x = rows(rate, [20000, 7000, 1], 3)
    x[1, 5] = -0.0
    for spec in ("mix=0", "rt60=2,mix=0", {"ir": user_ir(5 * rate, rate), "mix": 0.0}):
        y = eng.reverb(x, spec, rate, lengths=[20000, 7000, 1])
        assert np.array_equal(y.view(np.int32)[0], x.view(np.int32)[0]) and np.array_equal(y[1, :7000].view(np.int32),
                                                                                        x[1, :7000].view(np.int32))
        assert np.all(y[1, 7000:] == 0) and y[2, 0] == x[2, 0]
    for d in (0, 1, 511, 512, 700, 3000):
        ir = np.zeros(d + 1, np.float32)
        ir[d] = 1.0
        y = eng.reverb(x[0], {"ir": ir, "mix": 1.0}, rate)
        ref = np.concatenate([np.zeros(d), x[0, :x.shape[1] - d].astype(np.float64)])
        assert error_units(y, ref, x[0], ir, 1.0) <= TOL, d


def test_same_bits_in_every_mode_and_batch_position(eng):
    rate = 48000
    x = rows(rate, [5000, 3000, 70000, 6000], 1)
    base = eng.reverb(x, "hall", rate)
    try:
        for mode in ("fp32", "bf16x3", "fp16"):
            eng.set_precision(mode)
            assert np.array_equal(eng.reverb(x, "hall", rate), base), mode
    finally:
        eng.set_precision("bf16x3")
    for b in range(4):
        assert np.array_equal(eng.reverb(x[b], "hall", rate), base[b]), b
        perm = np.roll(np.arange(4), b)
        assert np.array_equal(eng.reverb(x[perm], "hall", rate), base[perm]), b


def test_forward_in_place(eng):
    rate = 44100
    x = rows(rate, [40000, 9000], 2)
    ref = eng.reverb(x, "hall", rate, lengths=[40000, 9000])
    x_t = torch.from_numpy(x).cuda()
    n_t = torch.tensor([40000, 9000], dtype=torch.int32, device="cuda")
    y_t = eng.reverb_forward(x_t, "hall", rate, lengths_t=n_t, out=x_t)
    assert y_t.data_ptr() == x_t.data_ptr()
    assert np.array_equal(y_t.cpu().numpy(), ref)
    ir = {"ir": user_ir(777, rate), "mix": 0.4}
    assert np.array_equal(eng.reverb_forward(torch.from_numpy(x).cuda(), ir, rate).cpu().numpy(), eng.reverb(x, ir, rate))


@pytest.mark.parametrize("S", [1, 3, 32])
@pytest.mark.parametrize("pattern,device", [("one", False), ("full", False), ("full", True), ("random", False), ("random", True)])
def test_stream_equals_one_shot(eng, S, pattern, device):
    """rows pushed in `pattern` chunks and held to the stream's contract on every push (tests/helpers/slot_streams.py)"""
    rate = 48000
    if pattern == "one" and S == 32:
        pytest.skip("one-sample pushes run at S = 1 and 3")
    lengths = [int(v) for v in np.random.default_rng(S).integers(1, 2500 if pattern == "one" else 30000, size=S)]
    x = rows(rate, lengths, S)
    rng = np.random.default_rng(7)
    for spec in ("hall", {"ir": user_ir(1500, rate), "mix": 0.7}):
        for chunk in (300, 1500):
            stage = ss.stage(eng, "reverb", S, chunk, rate, spec=spec)
            with stage.open() as st:
                assert st.lookahead == 511 and st.out_pitch == chunk + 511
            ss.run(stage, [[ss.pattern(pattern, n, chunk, rng)] for n in lengths], lambda s, u, n: x[s, :n], host=not device)
            if pattern == "one":
                break


def test_launch_counts(eng):
    rate = 16000
    x = rows(rate, [4000], 0)
    with eng.open_reverb_stream(1, 500, "hall", rate) as st:
        for i in range(8):
            c0 = eng.launch_count()
            st.push(x[:, 500 * i:500 * i + 500], [500], [i == 0], [i == 7])
            assert eng.launch_count() - c0 == 4
    with eng.open_reverb_stream(32, 3000, "room", rate) as st:
        c0 = eng.launch_count()
        st.push(np.zeros((32, 3000), np.float32), np.full(32, 3000), np.ones(32, bool), None)
        assert eng.launch_count() - c0 == 4
    for shape in ((3, 50000), (1, 10)):
        c0 = eng.launch_count()
        eng.reverb(np.zeros(shape, np.float32), "hall", rate)
        assert eng.launch_count() - c0 == 4


def test_argument_errors(eng):
    from viettts_b200 import _lib
    x = np.zeros((2, 100), np.float32)
    for spec in ("rt60=5", "mix=nan", "predelay=300", {"ir": [np.nan]}, {"ir": np.ones(80001)}):
        with pytest.raises(ValueError):
            eng.reverb(x, spec)
    with pytest.raises(ValueError):
        eng.reverb(x, "room", lengths=[1, 2, 3])
    lib = eng.lib
    y = np.zeros_like(x)
    ir = np.ones(40001, np.float32)
    c0 = eng.launch_count()
    for rate, L, mix in ((16000, 0, 0.5), (8000, 40001, 0.5), (16000, 10, float("nan")), (16000, 10, -0.1), (16000, 10, 1.5),
                         (7999, 10, 0.5), (192001, 10, 0.5)):
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_reverb_host(eng.h, x.ctypes.data, None, 2, 100, rate, ir.ctypes.data, L, mix, y.ctypes.data))
    bad = ir.copy()
    bad[7] = np.nan
    with pytest.raises(_lib.VttsError, match="ir"):
        eng._ck(lib.vtts_reverb_host(eng.h, x.ctypes.data, None, 2, 100, 16000, bad.ctypes.data, 10, 0.5, y.ctypes.data))
    for B, S in ((0, 100), (2, 0)):
        with pytest.raises(_lib.VttsError):
            eng._ck(lib.vtts_reverb_host(eng.h, x.ctypes.data, None, B, S, 16000, ir.ctypes.data, 10, 0.5, y.ctypes.data))
    n = np.array([5, 200], np.int32)
    with pytest.raises(_lib.VttsError, match="outside"):
        eng._ck(lib.vtts_reverb_host(eng.h, x.ctypes.data, n.ctypes.data, 2, 100, 16000, ir.ctypes.data, 10, 0.5, y.ctypes.data))
    h, p = ctypes.c_void_p(), ctypes.c_int()
    with pytest.raises(_lib.VttsError, match="L="):
        eng._ck(lib.vtts_reverb_stream_create(eng.h, 2, 64, 8000, ir.ctypes.data, 40001, 0.5, ctypes.byref(h), ctypes.byref(p)))
    with pytest.raises(_lib.VttsError, match="ir"):
        eng._ck(lib.vtts_reverb_stream_create(eng.h, 2, 64, 16000, bad.ctypes.data, 10, 0.5, ctypes.byref(h), ctypes.byref(p)))
    with pytest.raises(_lib.VttsError, match="max_streams"):
        eng._ck(lib.vtts_reverb_stream_create(eng.h, 0, 64, 16000, ir.ctypes.data, 10, 0.5, ctypes.byref(h), ctypes.byref(p)))
    assert eng.launch_count() == c0
    with eng.open_reverb_stream(2, 64) as st:
        c0 = eng.launch_count()
        with pytest.raises(_lib.VttsError, match="not open"):
            st.push(np.zeros((2, 64), np.float32), [64, 0], None, None)
        with pytest.raises(_lib.VttsError, match="outside"):
            st.push(np.zeros((2, 64), np.float32), [65, 0], [True, False], None)
        with pytest.raises(ValueError):
            st.push(np.zeros((2, 65), np.float32), [64, 0], [True, False], None)
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


@pytest.mark.parametrize("rate,deess,limit", [(None, None, None), (None, "threshold=-50", -1.0), (48000, None, None),
                                              (48000, "voice", -3.0)])
def test_tts_stream_reverb(tts_eng, rate, deess, limit):
    from viettts_b200.engine import AudioChain
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(170 + b, n) for b, n in enumerate([25, 40])]
        audio = {0: [], 1: []}
        spec = "rt60=0.8,mix=0.3"
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, deess=deess, reverb=spec, limit=limit) as ts:
            assert ts.rv is not None and ts.rv.lookahead == 511
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
        chain = AudioChain(output_rate=rate, deess=deess, reverb=spec, limit=limit)
        for s in (0, 1):
            w = chain.run(eng, eng.tts(toks[s][None], silence_duration=0.1)[0][0])
            assert np.array_equal(np.concatenate(audio[s]), w), s
        with pytest.raises(ValueError, match="reverb"):
            eng.open_tts_stream(1, 16, 2000, 100, reverb="rt60=9")
    finally:
        eng.set_fused_pairs(True)


def test_cli_reverb(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
                             "--reverb", "room"]) == 0
    expect = synthesizer.float_to_pcm16(ge.reverb(wave, "room", 16000)).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
    assert synthesizer.main(["--text", text, "--output", "two.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--output-rate", "48000", "--reverb", "hall", "--limiter"]) == 0
    r = ge.reverb(ge.resample(wave, 48000), "hall", 48000)
    expect = synthesizer.float_to_pcm16(ge.limit(r, -1.0, 48000)[0]).astype(np.int32)
    raw = np.frombuffer((tmp_path / "two.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1
