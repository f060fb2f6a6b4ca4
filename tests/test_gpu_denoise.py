"""GPU: the bias denoiser (Engine.denoise / denoise_forward / denoiser_bias, vtts_denoise*), its stream
(Engine.open_denoise_stream) and the `denoise=` strength of the text-to-speech stream and the CLI.

One-shot outputs are held to the float64 definition per element, |y - y64| <= TOL * error_scale (TOL from
tests/test_denoise_cpu.py, over 4x an fp32 emulation of the kernels); everything that streams, and every precision mode,
batch position and repeat, is compared bit for bit (np.array_equal) with the one-shot call."""
import ctypes as C
import json
import pickle

import numpy as np
import pytest
import torch

from helpers import slot_streams as ss
from oracle import denoise_oracle as do
from test_denoise_cpu import STRENGTHS, TOL, hiss_bias, signal_of
from viettts_b200 import config, synthetic

pytestmark = pytest.mark.gpu
KEY = np.array([7, 1234567], np.uint32)
RAGGED = [0, 1, 511, 512, 513, 767, 1023, 1024, 1025, 80128]


@pytest.fixture(scope="module")
def eng():
    from viettts_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def check_row(y, x, n, s, bias, what=""):
    """y: the full output row of an input row x of which n samples are valid"""
    if n <= do.PAD:
        assert np.array_equal(y[:n].view(np.uint32), x[:n].view(np.uint32)), what     # short rows: a bit copy
    else:
        y64 = do.denoise(x[:n], s, bias)
        scale = do.error_scale(x[:n], s, bias)
        ratio = np.abs(y[:n].astype(np.float64) - y64) / scale
        assert np.all(ratio <= TOL), (what, float(ratio.max()))
    assert np.all(y[n:] == 0), what


@pytest.mark.parametrize("s", STRENGTHS)
def test_one_shot_ragged_batch_against_float64(eng, s):
    bias = hiss_bias()
    S = max(RAGGED)
    lens = np.array(RAGGED, np.int32)
    x = np.stack([signal_of(S, 40 + b) for b in range(lens.size)])
    for b, n in enumerate(lens):
        x[b, n:] = np.nan                             # past a row's length: never read
    y = eng.denoise(x, s, lengths=lens, bias=bias)
    assert y.shape == x.shape
    for b, n in enumerate(lens):
        check_row(y[b], x[b], int(n), s, bias, (s, b, n))
    # the device entry point computes the same bits
    dev = torch.device("cuda", 0)
    yt = eng.denoise_forward(torch.from_numpy(x).to(dev), s, lengths_t=torch.from_numpy(lens).to(dev),
                             bias_t=torch.from_numpy(bias).to(dev))
    assert np.array_equal(yt.cpu().numpy(), y)


def test_three_minute_row(eng):
    n = 3 * 60 * 16000 + 77
    x = signal_of(n, 11)
    bias = hiss_bias()
    y = eng.denoise(x, 0.1, bias=bias)
    check_row(y, x, n, 0.1, bias, "3 min")


def test_same_bits_in_every_mode_alone_in_a_batch_and_repeated(eng):
    bias = hiss_bias()
    S = 20000
    lens = np.array([S, 7000, 513, 300], np.int32)
    x = np.stack([signal_of(S, 60 + b) for b in range(lens.size)])
    ys = []
    for mode in ("fp32", "bf16x3", "fp16"):
        eng.set_precision(mode)
        ys.append(eng.denoise(x, 0.5, lengths=lens, bias=bias))
        ys.append(eng.denoise(x, 0.5, lengths=lens, bias=bias))
    eng.set_precision("bf16x3")
    for y in ys[1:]:
        assert np.array_equal(y, ys[0])
    for b, n in enumerate(lens):
        alone = eng.denoise(x[b, :n], 0.5, bias=bias)
        assert np.array_equal(alone, ys[0][b, :n]), b


def test_zero_strength_reconstructs(eng):
    x = signal_of(9000, 3)
    y = eng.denoise(x, 0.0, bias=hiss_bias())
    assert np.abs(y - x).max() <= 1e-5


# ---- stream ------------------------------------------------------------------------------------------------------

KINDS = [k for k in ss.KINDS if k != "late"]


def run_stream(eng, S, F, kinds, strength, seed):
    """slot s runs plan kinds[s]; every push is held to the stream's contract (tests/helpers/slot_streams.py)"""
    rng = np.random.default_rng(seed)
    stage = ss.stage(eng, "denoise", S, F, strength=strength, bias=hiss_bias())
    with stage.open() as ds:
        assert ds.lookahead == do.LOOKAHEAD
    ss.run(stage, [ss.push_plan(k, F, rng) for k in kinds], lambda s, u, n: signal_of(n, 1000 * s + u))


@pytest.mark.parametrize("S", [1, 3, 32])
def test_stream_equals_one_shot(eng, S):
    kinds = ["max"] if S == 1 else [KINDS[(s + S) % len(KINDS)] for s in range(S)]
    run_stream(eng, S, 1000, kinds, 0.3, seed=S)


def test_stream_one_sample_pushes_and_edges(eng):
    run_stream(eng, 4, 1024, ["ones", 255, 256, "short"], 1.0, seed=99)


def test_stream_host_push_equals_device_push(eng):
    F = 700
    x = signal_of(5000, 4)
    bias = hiss_bias()
    with eng.open_denoise_stream(2, F, 0.2, bias=bias) as ds:
        out = [[], []]
        for p0 in range(0, 5000, F):
            n = min(F, 5000 - p0)
            ys = ds.push(np.stack([x[p0: p0 + n], -x[p0: p0 + n]]), [n, n], begin=[p0 == 0] * 2, end=[p0 + n == 5000] * 2)
            for s in range(2):
                out[s].append(ys[s])
    ref = eng.denoise(np.stack([x, -x]), 0.2, bias=bias)
    for s in range(2):
        assert np.array_equal(np.concatenate(out[s]), ref[s])


def test_launches_are_fixed(eng):
    with eng.open_denoise_stream(4, 512, 0.1, bias=hiss_bias()) as ds:
        counts = []
        for n_new, flags in (([0, 0, 0, 0], [0, 0, 0, 0]), ([512, 1, 0, 7], [1, 1, 0, 3]), ([512, 0, 0, 0], [0, 2, 0, 0]),
                             ([0, 0, 0, 0], [0, 0, 0, 0])):
            before = eng.launch_count()
            ds.push(np.zeros((4, 512), np.float32), n_new, begin=np.array(flags) & 1, end=np.array(flags) & 2)
            counts.append(eng.launch_count() - before)
    assert counts == [3, 3, 3, 3]
    before = eng.launch_count()
    eng.denoise(np.zeros((3, 1000), np.float32), 0.1, bias=hiss_bias())
    assert eng.launch_count() - before == 2


def test_argument_errors(eng):
    from viettts_b200._lib import VttsError
    x = signal_of(2000, 1)
    bias = hiss_bias()
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            eng.denoise(x, bad, bias=bias)
        with pytest.raises(ValueError):
            eng.open_denoise_stream(1, 16, bad, bias=bias)
        # the library checks too
        assert eng.lib.vtts_denoise_host(eng.h, x.ctypes.data, None, 1, x.size, bad, bias.ctypes.data, x.ctypes.data) == -1
    for b in (np.full(513, -1.0, np.float32), np.full(513, np.nan, np.float32)):
        with pytest.raises(ValueError):
            eng.denoise(x, 0.1, bias=b)
        assert eng.lib.vtts_denoise_host(eng.h, x.ctypes.data, None, 1, x.size, 0.1, b.ctypes.data, x.ctypes.data) == -1
        h, pitch = C.c_void_p(), C.c_int()
        assert eng.lib.vtts_denoise_stream_create(eng.h, 1, 16, 0.1, b.ctypes.data, C.byref(h), C.byref(pitch)) == -1
    with pytest.raises(VttsError, match="outside"):
        eng.denoise(np.stack([x, x]), 0.1, lengths=[2000, 2001], bias=bias)
    with pytest.raises(VttsError, match="outside"):
        eng.denoise(np.stack([x, x]), 0.1, lengths=[-1, 5], bias=bias)
    xt = torch.from_numpy(x[None]).cuda()
    assert eng.lib.vtts_denoise(eng.h, xt.data_ptr(), None, 1, x.size, 0.1, torch.from_numpy(bias).cuda().data_ptr(), xt.data_ptr(),
                                None) == -1                                     # y aliases x
    for S, F in ((0, 16), (65536, 16), (1, 0), (1, (1 << 22) + 1)):
        with pytest.raises(VttsError, match="denoise_stream_create"):
            eng.open_denoise_stream(S, F, 0.1, bias=bias)
    with eng.open_denoise_stream(2, 16, 0.1, bias=bias) as ds:
        z = np.zeros((2, 16), np.float32)
        with pytest.raises(VttsError, match="not open"):
            ds.push(z, [4, 0])
        with pytest.raises(VttsError, match="outside"):
            ds.push(z, [17, 0], begin=[True, False])
        with pytest.raises(VttsError, match="flags"):
            ds.push_device(torch.zeros((2, 16), device="cuda"), [1, 0], np.array([4, 0], np.uint8),
                           torch.zeros((2, ds.out_pitch), device="cuda"))
        ds.push(z, [4, 0], begin=[True, False], end=[True, False])
        with pytest.raises(VttsError, match="not open"):
            ds.push(z, [4, 0])                        # ended: BEGIN first
        y = ds.push(np.stack([x[:16], x[:16]]), [16, 0], begin=[True, False], end=[True, False])[0]
        assert np.array_equal(y, x[:16])              # a short row is a copy, and the failed calls left the stream usable


# ---- default bias, text-to-speech stream and CLI -------------------------------------------------------------

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


def check_bias(beta, wav, what):
    """beta against |X_0| of wav in float64; a bin's rounding error scales with the spectrum's norm, which is 32 times the
    windowed frame's (Parseval, N = 1024)"""
    b64 = do.bias_of(wav)
    scale = 32 * np.linalg.norm(do.frames(wav)[0] * do.window())
    assert beta.shape == (do.N_BINS,) and np.all(beta >= 0), what
    assert np.abs(beta - b64).max() <= TOL * scale, (what, float(np.abs(beta - b64).max() / scale))


def test_denoiser_bias_is_frame0_of_the_zero_mel_output(tts_eng):
    eng = tts_eng
    mel = np.random.default_rng(3).standard_normal((40, config.MEL_DIM)).astype(np.float32)
    for mode in ("bf16x3", "fp16", "fp32"):
        eng.set_precision(mode)
        beta = eng.denoiser_bias()
        check_bias(beta, eng.mel2wave(np.zeros((1, do.ZERO_MEL_FRAMES, config.MEL_DIM), np.float32))[0], mode)
        assert np.array_equal(eng.denoiser_bias(), beta)            # cached until the mode or the generator changes
        check_bias(eng.denoiser_bias(mel), eng.mel2wave(mel[None])[0], (mode, "mel"))
    eng.set_precision("bf16x3")


@pytest.mark.parametrize("kind", ["off", "reference"])
@pytest.mark.parametrize("rate", [None, 48000])
def test_tts_stream_denoise_equals_denoised_tts(tts_eng, rate, kind):
    eng = tts_eng
    eng.set_precision("bf16x3")
    eng.set_fused_pairs(False)
    try:
        strength = 0.5
        lens = [30, 7, 55, 20]
        kw = {"off": {}, "reference": {"rng": KEY}}[kind]
        toks = [tts_tokens(80 + b, n) for b, n in enumerate(lens)]
        expect = []
        for t in toks:
            w = eng.denoise(eng.tts(t[None], silence_duration=0.1, **kw)[0][0], strength)
            expect.append(w if rate is None else eng.resample(w, rate))
        pieces = {b: [] for b in range(len(toks))}
        with eng.open_tts_stream(2, 16, 2000, 100, output_rate=rate, denoise=strength, **kw) as ts:
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


def test_cli_denoise(tts_eng, acoustic_ckpt, hifigan_params, golden_dir, tmp_path, monkeypatch):
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
                             "--denoise", "0.3"]) == 0
    wave = np.ravel(mel2wave(text2mel(synthesizer.nat_normalize_text(text), lex, 0.1)))
    raw = (tmp_path / "one.wav").read_bytes()
    assert synthesizer.read_wav(tmp_path / "one.wav")[1] == 16000
    assert raw[44:] == synthesizer.float_to_pcm16(ge.denoise(wave, 0.3)).tobytes()

    lines = ["Xin chào, tôi là trợ lý ảo.", "hôm nay trời đẹp quá! bạn có khỏe không?"]
    (tmp_path / "lines.txt").write_text("\n".join(lines) + "\n")
    assert synthesizer.main(["--text-file", "lines.txt", "--output", "out.wav", "--lexicon-file", lex, "--silence-duration", "0.1",
                             "--seed", "5", "--denoise", "0.3", "--output-rate", "48000"]) == 0
    waves = synthesizer.synthesize_lines(lines, lex, 0.1, seed=5)
    for i, w in enumerate(waves):
        raw = (tmp_path / f"out_{i:04d}.wav").read_bytes()
        assert synthesizer.read_wav(tmp_path / f"out_{i:04d}.wav")[1] == 48000
        assert raw[44:] == synthesizer.float_to_pcm16(ge.resample(ge.denoise(w, 0.3), 48000)).tobytes()

    with pytest.raises(SystemExit):
        synthesizer.main(["--text", text, "--denoise", "-0.5", "--lexicon-file", lex])
