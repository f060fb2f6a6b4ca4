"""GPU: the resampler (Engine.resample / resample_forward, vtts_resample*), its stream (Engine.open_resample_stream) and
the output rate of the text-to-speech stream and the CLI.

One-shot outputs are held to the float64 definition per element, |y - y64| <= TOL * sum|h x| (TOL from
tests/test_resample_cpu.py, 4x over an emulation of the kernel's fp32 sum order); everything that streams is compared
bit for bit (np.array_equal) with the one-shot call."""
import json
import pickle

import numpy as np
import pytest
import torch

from oracle import resample_oracle as ro
from test_resample_cpu import LENGTHS, RATES, SR, TOL, signal_of
from viettts_b200 import config, synthetic
from viettts_b200.engine import STREAM_BEGIN, STREAM_END

pytestmark = pytest.mark.gpu
STREAM_RATES = [(SR, 48000), (SR, 44100), (SR, 11025), (SR, 8000), (48000, SR)]
KEY = np.array([7, 1234567], np.uint32)


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def check_row(y, x, n, rates, what=""):
    """y: the full output row of an input row x of which n samples are valid"""
    n_out = ro.out_len(n, *rates)
    if n > 0:
        y64 = ro.resample(x[:n], *rates)
        scale = ro.abs_sum(x[:n], *rates)
        err = np.abs(y[:n_out].astype(np.float64) - y64)
        assert np.all(err <= TOL * scale), (what, float((err / np.maximum(scale, 1e-30)).max()))
    assert np.all(y[n_out:] == 0), what


@pytest.mark.parametrize("rates", RATES, ids=lambda r: f"{r[0]}-{r[1]}")
def test_one_shot_against_float64(eng, rates):
    for n in LENGTHS:
        x = signal_of(n, n)
        y = eng.resample(x, rates[1], in_rate=rates[0])
        assert y.shape == (ro.out_len(n, *rates),)
        check_row(y, x, n, rates, n)
    # ragged batch: samples past a row's length are NaN and must not be read; outputs past its length are 0
    S = 3000
    lens = np.array([S, 1, 257, 2999, 0, 1500], np.int32)
    x = np.stack([signal_of(S, 50 + b) for b in range(lens.size)])
    for b, n in enumerate(lens):
        x[b, n:] = np.nan
    y = eng.resample(x, rates[1], in_rate=rates[0], lengths=lens)
    assert y.shape == (lens.size, ro.out_len(S, *rates))
    for b, n in enumerate(lens):
        check_row(y[b], x[b], int(n), rates, (b, n))
    # the device entry point computes the same bits
    dev = torch.device("cuda", 0)
    yt = eng.resample_forward(torch.from_numpy(x).to(dev), rates[1], in_rate=rates[0], lengths_t=torch.from_numpy(lens).to(dev))
    assert np.array_equal(yt.cpu().numpy(), y)


def test_same_rate_is_a_bit_copy(eng):
    x = signal_of(4097, 1)
    x[::7] = -0.0
    x[3] = 1e-40                      # a subnormal survives
    y = eng.resample(x, SR)
    assert np.array_equal(y.view(np.uint32), x.view(np.uint32))


def test_precision_mode_does_not_matter(eng):
    x = signal_of(5000, 2)
    ys = []
    for mode in ("fp32", "bf16x3", "fp16"):
        eng.set_precision(mode)
        ys.append(eng.resample(x, 44100))
    eng.set_precision("bf16x3")
    assert np.array_equal(ys[0], ys[1]) and np.array_equal(ys[0], ys[2])


LONG = 5_000_000 + 12_345


@pytest.fixture(scope="module")
def long_row():
    """16000 -> 11025 over more than 5 M samples: its last outputs have m * down + half >= 2^31"""
    rates = (SR, 11025)
    x = signal_of(LONG, 9)
    up, down, half = ro.ratio(*rates)
    n_out = ro.out_len(LONG, *rates)
    assert (n_out - 1) * down + half >= 2 ** 31
    return rates, x


def test_long_row_64bit_indices(eng, long_row):
    rates, x = long_row
    y = eng.resample(x, rates[1], in_rate=rates[0])
    n_out = y.size
    m0 = n_out - 4000
    y64 = ro.resample(x, *rates, m_range=(m0, n_out))
    scale = ro.abs_sum(x, *rates, m_range=(m0, n_out))
    assert np.all(np.abs(y[m0:] - y64) <= TOL * scale)
    # and a window in the middle, where the index first passes 2^31
    up, down, half = ro.ratio(*rates)
    mc = (2 ** 31 - half) // down
    y64 = ro.resample(x, *rates, m_range=(mc - 500, mc + 500))
    scale = ro.abs_sum(x, *rates, m_range=(mc - 500, mc + 500))
    assert np.all(np.abs(y[mc - 500: mc + 500] - y64) <= TOL * scale)


def test_long_row_streams_in_max_size_pushes(eng, long_row):
    rates, x = long_row
    ref = eng.resample(x, rates[1], in_rate=rates[0])
    F = 1 << 18
    dev = torch.device("cuda", 0)
    out = []
    with eng.open_resample_stream(1, F, rates[1], in_rate=rates[0]) as rs:
        xt = torch.zeros((1, F), device=dev)
        yt = torch.zeros((1, rs.out_pitch), device=dev)
        for p0 in range(0, LONG, F):
            n = min(F, LONG - p0)
            xt[0, :n] = torch.from_numpy(x[p0: p0 + n]).to(dev)
            flags = np.array([(STREAM_BEGIN if p0 == 0 else 0) | (STREAM_END if p0 + n == LONG else 0)], np.uint8)
            k = rs.push_device(xt, [n], flags, yt)
            out.append(yt[0, : int(k[0])].cpu().numpy())
    assert np.array_equal(np.concatenate(out), ref)


# ---- stream ------------------------------------------------------------------------------------------------------

def slot_plan(kind, s, F, D, rng):
    """list of utterances, each a list of (n_new, flags) pushes, for slot s; 'rebegin' starts a second utterance over an
    open first one"""
    def sizes(total, pick):
        out, left = [], total
        while left > 0:
            n = min(left, pick())
            out.append(n)
            left -= n
        return out

    if kind == "ones":
        pushes = [[1] * int(rng.integers(30, 80))]
    elif kind == "edges":
        cyc = [max(1, D - 1), max(1, D), min(F, 256), F]
        pushes = [sizes(int(rng.integers(2 * F, 4 * F)), lambda it=iter(cyc * 100): next(it))]
    elif kind == "random":
        pushes = [[int(v) for v in rng.integers(0, F + 1, size=int(rng.integers(3, 12)))]]
    elif kind == "single":
        pushes = [[int(rng.integers(1, F + 1))]]
    elif kind == "end_empty":
        pushes = [[int(v) for v in rng.integers(1, F + 1, size=3)] + [0]]
    elif kind == "reuse":
        pushes = [[int(v) for v in rng.integers(1, F + 1, size=3)], [int(v) for v in rng.integers(1, F + 1, size=2)]]
    elif kind == "rebegin":
        pushes = [[int(v) for v in rng.integers(1, F + 1, size=2)], [int(v) for v in rng.integers(1, F + 1, size=3)]]
    else:   # idle: never pushed
        pushes = []
    plan = []
    for u, p in enumerate(pushes):
        if kind == "random":
            p[0] = max(1, p[0])
        for q, n in enumerate(p):
            f = (STREAM_BEGIN if q == 0 else 0)
            if q == len(p) - 1 and not (kind == "rebegin" and u == 0):
                f |= STREAM_END
            if n == 0 and f == 0:
                plan.append((0, 0, u))       # an idle push inside the utterance
            else:
                plan.append((n, f, u))
    return plan


KINDS = ["ones", "edges", "random", "single", "end_empty", "reuse", "rebegin", "idle"]


@pytest.mark.parametrize("S", [1, 8, 33])
@pytest.mark.parametrize("rates", STREAM_RATES, ids=lambda r: f"{r[0]}-{r[1]}")
def test_stream_equals_one_shot(eng, rates, S):
    F = 1024
    rng = np.random.default_rng(S * 7 + rates[1])
    dev = torch.device("cuda", 0)
    with eng.open_resample_stream(S, F, rates[1], in_rate=rates[0]) as rs:
        D = rs.lookahead
        assert D == ro.lookahead(*rates)
        kinds = [KINDS[(s + (0 if S > 1 else 1)) % len(KINDS)] for s in range(S)] if S > 1 else ["edges"]
        plans = [slot_plan(k, s, F, D, rng) for s, k in enumerate(kinds)]
        # per slot and utterance: the input samples, the outputs received
        data = [dict() for _ in range(S)]
        got = [dict() for _ in range(S)]
        P = np.zeros(S, np.int64)
        E = np.zeros(S, np.int64)
        xt = torch.zeros((S, F), device=dev)
        yt = torch.empty((S, rs.out_pitch), device=dev)
        for c in range(max(len(p) for p in plans)):
            n_new = np.zeros(S, np.int32)
            flags = np.zeros(S, np.uint8)
            x = np.zeros((S, F), np.float32)
            for s in range(S):
                if c >= len(plans[s]):
                    continue
                n, f, u = plans[s][c]
                n_new[s], flags[s] = n, f
                chunk = signal_of(n, 1000 * s + 10 * c + u) if n else np.zeros(0, np.float32)
                x[s, :n] = chunk
                x[s, n:] = np.nan                         # past n_new: never read
                if f & STREAM_BEGIN:
                    data[s][u], got[s][u] = [], []
                    P[s] = E[s] = 0
                if n or f:
                    data[s][u].append(chunk)
            xt.copy_(torch.from_numpy(x))
            yt.fill_(12345.0)
            before = eng.launch_count()
            n_out = rs.push_device(xt, n_new, flags, yt)
            assert eng.launch_count() - before == 2
            y = yt.cpu().numpy()
            for s in range(S):
                active = n_new[s] > 0 or flags[s] != 0
                if not active:
                    assert n_out[s] == 0 and np.all(y[s] == 12345.0), (s, c)     # idle: untouched
                    continue
                P[s] += n_new[s]
                e = ro.out_len(int(P[s]), *rates) if flags[s] & STREAM_END else ro.emitted_closed_form(int(P[s]), *rates)
                assert n_out[s] == e - E[s], (kinds[s], s, c, int(P[s]), int(n_out[s]), e - E[s])
                E[s] = e
                got[s][plans[s][c][2]].append(y[s, : n_out[s]].copy())
        for s in range(S):
            for u, chunks in data[s].items():
                xs = np.concatenate(chunks) if chunks else np.zeros(0, np.float32)
                out = np.concatenate(got[s][u]) if got[s][u] else np.zeros(0, np.float32)
                if kinds[s] == "rebegin" and u == 0:
                    # abandoned by the second BEGIN: what it emitted is the start of the one-shot result
                    ref = eng.resample(xs, rates[1], in_rate=rates[0]) if xs.size else np.zeros(0, np.float32)
                    assert np.array_equal(out, ref[: out.size]) and out.size == ro.emitted_closed_form(xs.size, *rates)
                    continue
                ref = eng.resample(xs, rates[1], in_rate=rates[0]) if xs.size else np.zeros(0, np.float32)
                assert out.shape == ref.shape and np.array_equal(out, ref), (kinds[s], s, u)


def test_stream_host_push_equals_device_push(eng):
    rates = (SR, 44100)
    F = 300
    x = signal_of(1000, 4)
    with eng.open_resample_stream(2, F, rates[1]) as rs:
        out = [[], []]
        for p0 in range(0, 1000, F):
            n = min(F, 1000 - p0)
            chunk = np.stack([x[p0: p0 + n], -x[p0: p0 + n]])
            ys = rs.push(chunk, [n, n], begin=[p0 == 0] * 2, end=[p0 + n == 1000] * 2)
            for s in range(2):
                out[s].append(ys[s])
    ref = eng.resample(np.stack([x, -x]), rates[1])
    for s in range(2):
        assert np.array_equal(np.concatenate(out[s]), ref[s])


def test_stream_launches_per_push_are_fixed(eng):
    with eng.open_resample_stream(4, 512, 48000) as rs:
        counts = []
        for n_new, flags in (([0, 0, 0, 0], [0, 0, 0, 0]), ([512, 1, 0, 7], [1, 1, 0, 3]), ([512, 0, 0, 0], [0, 2, 0, 0]),
                             ([0, 0, 0, 0], [0, 0, 0, 0])):
            before = eng.launch_count()
            rs.push(np.zeros((4, 512), np.float32), n_new, begin=np.array(flags) & 1, end=np.array(flags) & 2)
            counts.append(eng.launch_count() - before)
    assert counts == [2, 2, 2, 2]
    before = eng.launch_count()
    eng.resample(np.zeros((3, 1000), np.float32), 48000)
    assert eng.launch_count() - before == 1


def test_argument_errors(eng):
    from viettts_b200._lib import VttsError
    x = np.zeros(100, np.float32)
    for bad in (1031, 16001 * 1031):
        with pytest.raises(VttsError, match="reduced ratio"):
            eng.resample(x, bad)
        with pytest.raises(VttsError, match="reduced ratio"):
            eng.open_resample_stream(1, 16, bad)
    for bad in (0, -48000):
        with pytest.raises(ValueError):
            eng.resample(x, bad)
        with pytest.raises(ValueError):
            eng.open_resample_stream(1, 16, bad)
    assert eng.lib.vtts_resample_host(eng.h, x.ctypes.data, None, 1, 100, 0, 48000, x.ctypes.data) == -1
    assert eng.lib.vtts_resample_host(eng.h, x.ctypes.data, None, 0, 100, SR, 48000, x.ctypes.data) == -1
    assert eng.lib.vtts_resample_host(eng.h, x.ctypes.data, None, 1, 0, SR, 48000, x.ctypes.data) == -1
    for S, F in ((0, 16), (65536, 16), (1, 0), (1, (1 << 22) + 1)):
        with pytest.raises(VttsError, match="resample_stream_create"):
            eng.open_resample_stream(S, F, 48000)
    with eng.open_resample_stream(2, 16, 48000) as rs:
        z = np.zeros((2, 16), np.float32)
        with pytest.raises(VttsError, match="not open"):
            rs.push(z, [4, 0])
        with pytest.raises(VttsError, match="not open"):
            rs.push(z, [0, 0], end=[True, False])
        with pytest.raises(VttsError, match="outside"):
            rs.push(z, [17, 0], begin=[True, False])
        with pytest.raises(VttsError, match="outside"):
            rs.push(z, [-1, 0], begin=[True, False])
        with pytest.raises(VttsError, match="flags"):
            rs.push_device(torch.zeros((2, 16), device="cuda"), [1, 0], np.array([4, 0], np.uint8),
                           torch.zeros((2, rs.out_pitch), device="cuda"))
        with pytest.raises(ValueError):
            rs.push(np.zeros((2, 17), np.float32), [1, 0], begin=[True, False])
        rs.push(z, [4, 0], begin=[True, False], end=[True, False])
        with pytest.raises(VttsError, match="not open"):
            rs.push(z, [4, 0])                        # ended: BEGIN first
        # the failed calls left the stream usable
        x = signal_of(16, 5)
        y = rs.push(np.stack([x, x]), [16, 0], begin=[True, False], end=[True, False])[0]
        assert np.array_equal(y, eng.resample(x, 48000))


# ---- text-to-speech stream and CLI ---------------------------------------------------------------------------

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
@pytest.mark.parametrize("rate", [48000, 44100])
def test_tts_stream_output_rate_equals_resampled_tts(tts_eng, rate, kind):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        lens = [30, 7, 55, 20]
        kw = {"off": {}, "reference": {"rng": KEY}}[kind]
        toks = [tts_tokens(80 + b, n) for b, n in enumerate(lens)]
        expect = [eng.resample(eng.tts(t[None], silence_duration=0.1, **kw)[0][0], rate) for t in toks]
        pieces = {b: [] for b in range(len(toks))}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, **kw) as ts:
            queue, owner = list(range(len(toks))), {}
            while queue or ts.busy().any():
                for s in np.flatnonzero(~ts.busy()):
                    if queue:
                        b = queue.pop(0)
                        owner[int(s)] = b
                        ts.begin(int(s), toks[b], silence_duration=0.1)
                for s, w in ts.step().items():
                    pieces[owner[s]].append(w)
        for b in range(len(toks)):
            audio = np.concatenate(pieces[b])
            assert audio.shape == expect[b].shape and np.array_equal(audio, expect[b]), (rate, kind, b)
    finally:
        eng.set_fused_pairs(True)


def test_cli_output_rate(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
                             "--output-rate", "48000"]) == 0
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    raw = (tmp_path / "one.wav").read_bytes()
    _, sr = synthesizer.read_wav(tmp_path / "one.wav")
    assert sr == 48000
    assert raw[44:] == synthesizer.float_to_pcm16(ge.resample(wave, 48000)).tobytes()

    lines = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--seed", "5", "--output-rate", "48000", "--sample-rate", "48000"]) == 0
    waves = synthesizer.synthesize_lines(lines, lex, 0.1, seed=5)
    for i, w in enumerate(waves):
        raw = (tmp_path / f"out_{i:04d}.wav").read_bytes()
        _, sr = synthesizer.read_wav(tmp_path / f"out_{i:04d}.wav")
        assert sr == 48000
        assert raw[44:] == synthesizer.float_to_pcm16(ge.resample(w, 48000)).tobytes()

    for bad in (["--text", text, "--sample-rate", "22050", "--output-rate", "48000"], ["--text", text, "--output-rate", "16001"],
                ["--text-file", "lines.txt", "--sample-rate", "16000", "--output-rate", "8000"]):
        with pytest.raises(SystemExit):
            synthesizer.main(bad + ["--lexicon-file", lex])
