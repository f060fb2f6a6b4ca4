"""GPU: the time stretcher (Engine.time_stretch / time_stretch_forward, vtts_time_stretch*), its stream
(Engine.open_time_stretch_stream) and the `tempo=` stage of the text-to-speech stream and the CLI's --tempo.

One-shot outputs are held to the float64 definition under the device's own discrete decisions
(vtts_debug_time_stretch_decisions) per element, |y - y64| <= TOL * stretch_error_scale (TOL from
tests/test_time_stretch_cpu.py), and the device's decisions may differ from float64's only where float64's margin is
below DEC_MARGIN of the frame's norm.  Everything that streams, and every precision mode, batch position and repeat, is
compared bit for bit with the one-shot call."""
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import denoise_oracle as do
from oracle import time_stretch_oracle as tso
from test_denoise_cpu import signal_of
from test_pitch_cpu import voiced_of
from test_time_stretch_cpu import DEC_MARGIN, TOL, decision_margins
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu
KEY = np.array([7, 1234567], np.uint32)
RAGGED = [0, 1, 512, 513, 1023, 1025, 80128]
TEMPOS = [0.75, 1.25, 2.0, 0.5, 1.6180339, 1.0, 0.9]


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def decisions(eng, x, tempo, lens=None):
    dev = torch.device("cuda", 0)
    lt = None if lens is None else torch.from_numpy(np.asarray(lens, np.int32)).to(dev)
    return eng.debug_time_stretch_decisions(torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev), tempo, lt)


def check_row(y, x, n, a, dec, what=""):
    """y: the full output row of an input row x of which n samples are valid; dec: the device's decisions of the row"""
    M = tso.stretch_length(n, a)
    if n <= do.PAD or float(np.float32(a)) == 1.0:
        k = min(n, M)
        assert np.array_equal(y[:k].view(np.uint32), x[:k].view(np.uint32)), what     # a bit copy
        assert not y[k:M].any() and not dec.any(), what
    else:
        T = do.n_frames(M)
        assert not dec[T:].any(), what
        dec = dec[:T]
        flag_m, branch_m = decision_margins(x[:n], a)
        dec64 = tso.stretch_decisions_of(x[:n], a)
        f_dev, f64 = (dec & 1) == 1, (dec64 & 1) == 1
        assert np.all(flag_m[f_dev != f64] < DEC_MARGIN), what
        side = f_dev & f64 & ((dec >> 1 & 1) != (dec64 >> 1 & 1))
        assert np.all(branch_m[side] < DEC_MARGIN), what
        y64 = tso.time_stretch(x[:n], a, decisions=dec)
        ratio = np.abs(y[:M].astype(np.float64) - y64) / tso.stretch_error_scale(x[:n], a)
        assert np.all(ratio <= TOL), (what, float(ratio.max()), int(ratio.argmax()))
    assert np.all(y[M:] == 0), what


def test_one_shot_ragged_batch_against_float64(eng):
    S = max(RAGGED)
    lens = np.array(RAGGED, np.int32)
    x = np.stack([(voiced_of if b % 2 else signal_of)(S, 40 + b) for b in range(lens.size)])
    for b, n in enumerate(lens):
        x[b, n:] = np.nan                             # past a row's length: never read
    tp = np.array(TEMPOS, np.float32)
    y = eng.time_stretch(x, tp, lengths=lens)
    assert y.shape == (len(lens), max(tso.stretch_length(int(n), float(a)) for n, a in zip(lens, tp)))
    dec = decisions(eng, x, tp, lens)
    assert dec.shape == (len(lens), max(tso.stretch_length(S, float(a)) for a in tp) // do.HOP + 1, do.N_BINS)
    for b, n in enumerate(lens):
        check_row(y[b], x[b], int(n), float(tp[b]), dec[b], (b, n, tp[b]))
    # the device entry point computes the same bits, into a wider buffer sized from S
    dev = torch.device("cuda", 0)
    yt = eng.time_stretch_forward(torch.from_numpy(x).to(dev), tp, lengths_t=torch.from_numpy(lens).to(dev)).cpu().numpy()
    assert np.array_equal(yt[:, : y.shape[1]], y) and not yt[:, y.shape[1]:].any()
    for n, a in zip(lens, tp):
        assert eng.time_stretch_length(int(n), float(a)) == tso.stretch_length(int(n), float(a))


def test_three_minute_row(eng):
    n = 3 * 60 * 16000 + 77
    x = voiced_of(n, 11)
    y = eng.time_stretch(x, 1.25)
    check_row(y, x, n, 1.25, decisions(eng, x[None], 1.25)[0], "3 min")


def test_same_bits_in_every_mode_alone_in_a_batch_and_repeated(eng):
    S = 20000
    lens = np.array([S, 7000, 513, 300], np.int32)
    tp = np.array([0.75, 2.0, 0.5, 1.25], np.float32)
    x = np.stack([voiced_of(S, 60 + b) for b in range(lens.size)])
    ys = []
    for mode in ("fp32", "bf16x3", "fp16"):
        eng.set_precision(mode)
        ys.append(eng.time_stretch(x, tp, lengths=lens))
        ys.append(eng.time_stretch(x, tp, lengths=lens))
    eng.set_precision("bf16x3")
    for y in ys[1:]:
        assert np.array_equal(y, ys[0])
    for b, n in enumerate(lens):
        alone = eng.time_stretch(x[b, :n], float(tp[b]))
        assert np.array_equal(alone, ys[0][b, : alone.size]) and not ys[0][b, alone.size:].any(), b


def test_unit_tempo_is_the_input(eng):
    x = voiced_of(9000, 3)
    assert np.array_equal(eng.time_stretch(x, 1.0), x)
    y = eng.time_stretch(np.stack([x, x]), [1.0, 1.5])
    assert y.shape == (2, 9000) and np.array_equal(y[0], x) and not np.array_equal(y[1, :6000], x[:6000])


# ---- stream ------------------------------------------------------------------------------------------------------

STREAM_TEMPOS = [0.75, 1.25, 1.0, 2.0, 0.5, 1.37, 0.9]


def run_stream(eng, S, F, kinds, seed):
    """slot s runs plan kinds[s], every utterance at its own tempo, held to the stream's contract and the oracle's
    schedule on every push (tests/helpers/slot_streams.py); at tempo 1 the stream is the input"""
    rng = np.random.default_rng(seed)
    plans = [ss.push_plan(k, F, rng) for k in kinds]
    tempos = [[STREAM_TEMPOS[int(rng.integers(len(STREAM_TEMPOS)))] for _ in p] for p in plans]
    stage = ss.stage(eng, "time_stretch", S, F)
    with stage.open() as ts:
        assert ts.lookahead == tso.TS_LOOKAHEAD
    for row in ss.run(stage, plans, lambda s, u, n: voiced_of(n, 1000 * s + u), tempos):
        for x, tempo, y, _ in filter(None, row):
            if tempo == 1.0:
                assert np.array_equal(y, x)


@pytest.mark.parametrize("S", [1, 3, 32])
def test_stream_equals_one_shot(eng, S):
    kinds = ["max"] if S == 1 else [ss.KINDS[(s + S) % len(ss.KINDS)] for s in range(S)]
    run_stream(eng, S, 1000, kinds, seed=S)


def test_stream_one_sample_pushes_and_edges(eng):
    run_stream(eng, 4, 1024, ["ones", 255, 256, "short"], seed=99)


def test_stream_large_chunks(eng):
    run_stream(eng, 2, 48000, ["max", "reuse"], seed=7)


def test_stream_host_push_equals_device_push(eng):
    F = 700
    x = voiced_of(5000, 4)
    with eng.open_time_stretch_stream(2, F) as ts:
        out = [[], []]
        for p0 in range(0, 5000, F):
            n = min(F, 5000 - p0)
            ys = ts.push(np.stack([x[p0: p0 + n], -x[p0: p0 + n]]), [n, n], begin=[p0 == 0] * 2, end=[p0 + n == 5000] * 2,
                         tempo=[0.8, 1.7])
            for s in range(2):
                out[s].append(ys[s])
    for s, a in ((0, 0.8), (1, 1.7)):
        assert np.array_equal(np.concatenate(out[s]), eng.time_stretch(x if s == 0 else -x, a))


def test_launches_are_fixed(eng):
    with eng.open_time_stretch_stream(4, 512) as ts:
        counts = []
        for n_new, flags in (([0, 0, 0, 0], [0, 0, 0, 0]), ([512, 1, 0, 7], [1, 1, 0, 3]), ([512, 0, 0, 0], [0, 2, 0, 0]),
                             ([0, 0, 0, 0], [0, 0, 0, 0])):
            before = eng.launch_count()
            ts.push(np.zeros((4, 512), np.float32), n_new, begin=np.array(flags) & 1, end=np.array(flags) & 2, tempo=1.5)
            counts.append(eng.launch_count() - before)
    assert counts == [5, 5, 5, 5]
    before = eng.launch_count()
    eng.time_stretch(np.zeros((3, 1000), np.float32), 0.8)
    assert eng.launch_count() - before == 4


def test_argument_errors(eng):
    from viettts_b200._lib import VttsError
    x = voiced_of(2000, 1)
    y = np.zeros(4000, np.float32)
    for bad in (float("nan"), float("inf"), 0.49, 2.01, 0.0, -1.0):
        with pytest.raises(ValueError):
            eng.time_stretch(x, bad)
        # the library checks too, before anything is launched
        c0 = eng.launch_count()
        tp = np.array([bad], np.float32)
        assert eng.lib.vtts_time_stretch_host(eng.h, x.ctypes.data, None, 1, x.size, tp.ctypes.data, y.ctypes.data, 4000) == -1
        assert eng.lib.vtts_time_stretch_length(100, bad) == -1
        assert eng.launch_count() == c0
    assert eng.lib.vtts_time_stretch_length(-1, 1.0) == -1
    with pytest.raises(VttsError, match="outside"):
        eng.time_stretch(np.stack([x, x]), 1.5, lengths=[2000, 2001])
    with pytest.raises(ValueError):
        eng.time_stretch(np.stack([x, x]), [1.0, 1.2, 1.3])
    xt = torch.from_numpy(x[None]).cuda()
    tp = np.array([1.5], np.float32)
    c0 = eng.launch_count()
    assert eng.lib.vtts_time_stretch(eng.h, xt.data_ptr(), None, 1, x.size, tp.ctypes.data, xt.data_ptr(), 2000, None) == -1  # alias
    assert eng.lib.vtts_time_stretch(eng.h, xt.data_ptr(), None, 1, x.size, None, xt.data_ptr() + 4, 1000, None) == -1       # no tempo
    yt = torch.empty((1, 2000), device=xt.device)
    assert eng.lib.vtts_time_stretch(eng.h, xt.data_ptr(), None, 1, x.size, tp.ctypes.data, yt.data_ptr(), 0, None) == -1   # Sy = 0
    assert eng.lib.vtts_time_stretch(eng.h, xt.data_ptr(), None, 0, x.size, tp.ctypes.data, yt.data_ptr(), 2000, None) == -1  # B = 0
    assert eng.launch_count() == c0
    for S, F in ((0, 16), (65536, 16), (1, 0), (1, (1 << 22) + 1)):
        with pytest.raises(VttsError, match="time_stretch_stream_create"):
            eng.open_time_stretch_stream(S, F)
    with eng.open_time_stretch_stream(2, 16) as ts:
        z = np.zeros((2, 16), np.float32)
        c0 = eng.launch_count()
        with pytest.raises(VttsError, match="not open"):
            ts.push(z, [4, 0])
        with pytest.raises(VttsError, match="outside"):
            ts.push(z, [17, 0], begin=[True, False], tempo=1.5)
        for bad in (float("nan"), 2.5, 0.25):
            with pytest.raises(VttsError, match="tempo"):
                ts.push(z, [4, 0], begin=[True, False], tempo=[bad, 1.0])
        with pytest.raises(ValueError, match="tempo"):
            ts.push(z, [4, 0], begin=[True, False])
        assert eng.launch_count() == c0                                 # nothing was launched
        ts.push(z, [4, 0], begin=[True, False], tempo=[1.5, 1.0])
        c0 = eng.launch_count()
        n = np.array([4, 0], np.int32)
        f = np.zeros(2, np.uint8)
        for changed in (np.array([1.25, 1.0], np.float32), np.array([np.nan, 1.0], np.float32)):
            with pytest.raises(VttsError, match="until END"):
                eng._ck(eng.lib.vtts_time_stretch_stream_push_host(eng.h, ts.h, z.ctypes.data, n.ctypes.data, f.ctypes.data,
                                                                   changed.ctypes.data, np.zeros((2, ts.out_pitch), np.float32).ctypes.data,
                                                                   np.zeros(2, np.int32).ctypes.data))
        assert eng.launch_count() == c0
        ts.push(z, [4, 0], end=[True, False])
        with pytest.raises(VttsError, match="not open"):
            ts.push(z, [4, 0])                        # ended: BEGIN first
        y = ts.push(np.stack([x[:16], x[:16]]), [16, 0], begin=[True, False], end=[True, False], tempo=0.5)[0]
        assert np.array_equal(y[:16], x[:16]) and y.size == 32 and not y[16:].any()   # a short row is a copy


# ---- text-to-speech stream and CLI -------------------------------------------------------------------------------

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


@pytest.mark.parametrize("kind", ["off", "reference"])
@pytest.mark.parametrize("denoise,semitones,rate", [(None, None, None), (0.5, 3.0, 48000)])
def test_tts_stream_tempo_equals_stretched_tts(tts_eng, denoise, semitones, rate, kind):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        lens = [30, 7, 55, 20]
        tempos = [None, 0.5, None, 1.6]                                # None: the stream's default
        default = 1.25
        kw = {"off": {}, "reference": {"rng": KEY}}[kind]
        toks = [tts_tokens(90 + b, n) for b, n in enumerate(lens)]
        expect = []
        for t, tp in zip(toks, tempos):
            w = eng.tts(t[None], silence_duration=0.1, **kw)[0][0]
            if denoise is not None:
                w = eng.denoise(w, denoise)
            if semitones is not None:
                w = eng.pitch_shift(w, semitones)
            w = eng.time_stretch(w, default if tp is None else tp)
            expect.append(w if rate is None else eng.resample(w, rate))
        pieces = {b: [] for b in range(len(toks))}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, denoise=denoise, semitones=semitones, tempo=default, **kw) as ts:
            queue, owner = list(range(len(toks))), {}
            while queue or ts.busy().any():
                for s in np.flatnonzero(~ts.busy()):
                    if queue:
                        b = queue.pop(0)
                        owner[int(s)] = b
                        ts.begin(int(s), toks[b], silence_duration=0.1, tempo=tempos[b])
                for s, w in ts.step().items():
                    pieces[owner[s]].append(w)
        for b in range(len(toks)):
            audio = np.concatenate(pieces[b])
            assert audio.shape == expect[b].shape and np.array_equal(audio, expect[b]), (denoise, rate, kind, b)
    finally:
        eng.set_fused_pairs(True)


def test_tts_stream_tempo_with_meter(tts_eng):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        toks = [tts_tokens(120 + b, n) for b, n in enumerate([25, 40])]
        audio = {0: [], 1: []}
        last = {}
        with eng.open_tts_stream(2, 16, 2000, 100, tempo=0.5, meter=True) as ts:
            ts.begin(0, toks[0], silence_duration=0.1)
            ts.begin(1, toks[1], silence_duration=0.1, tempo=1.8)
            while ts.busy().any():
                for s, w in ts.step().items():
                    audio[s].append(w)
                last.update(ts.meter())
        for s, tp in ((0, 0.5), (1, 1.8)):
            a = np.concatenate(audio[s])
            assert np.array_equal(a, eng.time_stretch(eng.tts(toks[s][None], silence_duration=0.1)[0][0], tp)), s
            ref = eng.loudness(a)
            assert np.array_equal(np.array(last[s], np.float32), np.array(ref, np.float32)), s
        with pytest.raises(ValueError):
            eng.open_tts_stream(1, 16, 2000, 100, tempo=2.5)
        with eng.open_tts_stream(1, 16, 2000, 100) as ts:
            with pytest.raises(ValueError, match="tempo"):
                ts.begin(0, toks[0], tempo=1.2)
    finally:
        eng.set_fused_pairs(True)


def test_cli_tempo(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
    assert synthesizer.main(["--text", text, "--output", "one.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--tempo", "1.5"]) == 0
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    pcm, sr = synthesizer.read_wav(tmp_path / "one.wav")
    assert sr == 16000
    expect = synthesizer.float_to_pcm16(ge.time_stretch(wave, 1.5)).astype(np.int32)
    raw = np.frombuffer((tmp_path / "one.wav").read_bytes()[44:], "<i2").astype(np.int32)
    assert raw.shape == expect.shape and np.abs(raw - expect).max() <= 1

    lines = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--seed", "5", "--pitch", "-2.5", "--tempo", "0.8", "--output-rate", "48000"]) == 0
    waves = synthesizer.synthesize_lines(lines, lex, 0.1, seed=5)
    for i, w in enumerate(waves):
        raw = (tmp_path / f"out_{i:04d}.wav").read_bytes()
        assert raw[44:] == synthesizer.float_to_pcm16(ge.resample(ge.time_stretch(ge.pitch_shift(w, -2.5), 0.8), 48000)).tobytes()

    for bad in ("2.5", "nan", "0.4"):
        with pytest.raises(SystemExit):
            synthesizer.main(["--text", text, "--tempo", bad, "--lexicon-file", lex])
